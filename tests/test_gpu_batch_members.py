"""Members that join and leave a running batch (bb200_amcl_batch_add_member / _remove_member) on the GPU.  Every occupied
member equals, byte for byte, a standalone Amcl created when it joined and fed the same inputs: update results,
particles, weights and ancestors after every step, the estimates of update_clustered, and cluster estimates, histograms
and pose samples after kept and resampled steps.  A second batch that holds only the long-lived members and never
changes stays byte-identical to the churned one.  Also covered: the launches of a membership change and of a step after
churn, the vacant-slot rules, a new member's empty history, and validation."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
INVALID, STATE = -1, -4  # BB200_ERR_INVALID_ARGUMENT, BB200_ERR_STATE


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=14)


def motion(bb, k):
    return [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.OmnidirectionalDriveModelParam(*ALPHAS), bb.StationaryModelParam()][k % 3]


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


def odometry(scene, t, k):
    x, y, th = scene.poses[t - 1 if t % 5 == 4 else t]
    th = th + 0.01 * k
    return np.array([np.cos(th), np.sin(th), x + 0.02 * k, y])


def launches(batch, call):
    before = batch.launch_count()
    out = call()
    return batch.launch_count() - before, out


def measurement(bb, scene, t, k):
    """Points, a scan or a float32 cloud of the scene's scan t, by member."""
    pts = scene.scans[t % 12][: 150 + 3 * k]
    if k % 3 == 1:
        r = np.hypot(pts[:, 0], pts[:, 1]).astype(np.float32)
        return bb.LaserScan(r, np.float32(-np.pi / 2), np.float32(np.pi / (len(r) - 1)), 0.1, 30.0, 0)
    if k % 3 == 2:
        xyz = np.concatenate([pts, np.full((len(pts), 1), 0.5)], axis=1).astype(np.float32)
        return bb.PointCloud(xyz.tobytes(), 12, 0, np.float32, None, len(xyz))
    return pts


def feed_twin(bb, twin, pose, meas):
    if isinstance(meas, bb.LaserScan):
        return twin.update_scan(pose, meas.ranges, meas.angle_min, meas.angle_increment, meas.min_range, meas.max_range, meas.max_beams,
                                meas.laser_origin)
    if isinstance(meas, bb.PointCloud):
        return twin.update_point_cloud(pose, meas.data, meas.point_step, meas.x_offset, meas.dtype, meas.origin, meas.n_points)
    return twin.update(pose, meas)


def twin_histogram(bb, twin, linear, angular):
    import ctypes as C

    from beluga_b200 import _capi

    f = twin.filter
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, None, 0, C.byref(n), C.byref(top)) == 0
    bins = np.empty(max(n.value, 1), dtype=bb._CELL_DTYPE)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, bins.ctypes.data_as(C.POINTER(_capi.ClusterCell)), n.value,
                                                  C.byref(n), C.byref(top)) == 0
    return bins[:n.value], top.value


def assert_member_equals_twin(batch, m, twin, got, exp, where):
    assert result_bytes(got) == result_bytes(exp), where
    gs, gw = batch.particles(m)
    ts, tw = twin.particles()
    n = batch.member_size(m)
    assert n == len(ts), where
    assert gs[:n].tobytes() == ts.tobytes() and gw[:n].tobytes() == tw.tobytes(), where
    if exp.updated and exp.resampled and batch.params[m].record_ancestors:
        assert batch.ancestors(m).tobytes() == twin.filter.ancestors().tobytes(), where


def assert_published_equal(bb, batch, twins, step):
    """Cluster estimates, particle histograms and pose samples of every occupied member against its twin."""
    est = batch.cluster_estimates()
    hists = batch.particle_histograms(None, 0.05, 0.05)
    counts = [0 if q is None else min(700, q.max_particles) for q in batch.params]
    samples = batch.sample_states(counts, step)
    for m, twin in twins.items():
        tm, tc = twin.filter.cluster_estimate()
        assert est[m][0].tobytes() == tm.tobytes() and est[m][1].tobytes() == tc.tobytes(), m
        bins, top = hists[m]
        t_bins, t_top = twin_histogram(bb, twin, 0.05, 0.05)
        assert bins.tobytes() == t_bins.tobytes() and np.float64(top).tobytes() == np.float64(t_top).tobytes(), m
        assert samples[m].tobytes() == twin.filter.sample_states(counts[m], step).tobytes(), m
    for m, q in enumerate(batch.params):
        if q is None:
            assert est[m] is None and hists[m] is None and samples[m] is None


class Maps:
    """Three maps in one batch -- likelihood field, prob likelihood field, beam model -- and the twins' view of them."""

    def __init__(self, bb, scene):
        self.grid = bb.OccupancyGrid(scene.cells, scene.resolution)
        self.lfm = bb.LikelihoodFieldModelParam(**LFM)
        self.beam = bb.BeamModelParam(sigma_hit=0.2, lambda_short=0.1, beam_max_range=20.0)
        self.kinds = [(bb.SENSOR_LIKELIHOOD_FIELD, self.lfm), (bb.SENSOR_LIKELIHOOD_FIELD_PROB, self.lfm), (bb.SENSOR_BEAM, self.beam)]

    def add(self, bb, batch):
        return [batch.add_likelihood_field_map(self.lfm, self.grid), batch.add_likelihood_field_map(self.lfm, self.grid, prob=True),
                batch.add_beam_map(self.beam, self.grid)]

    def assign(self, batch, ids, m, twin, which):
        batch.update_map(m, ids[which])
        sensor, params = self.kinds[which]
        twin.update_map(sensor, params, self.grid)


def params_of(bb, kind, seed, **extra):
    """fixed: 2000 particles; kld: 500..2000; selective: 2000, selective resampling; keep: 1500 that never resample."""
    table = dict(fixed=dict(min_particles=2000, max_particles=2000), kld=dict(min_particles=500, max_particles=2000),
                 selective=dict(min_particles=2000, max_particles=2000, selective_resampling=True),
                 keep=dict(min_particles=1500, max_particles=1500, resample_interval=1000))
    return bb.AmclParams(seed=seed, resample_scheme=seed % 2, **table[kind], **extra)


def test_churn_against_twins_and_an_unchanged_batch(bb, scene):
    maps = Maps(bb, scene)
    # slot: (kind, map); slots 1, 3, 4 and 6 live throughout, the others leave and are replaced
    initial = [("fixed", 0), ("kld", 1), ("keep", 0), ("selective", 2), ("keep", 1), ("kld", 0), ("selective", 0), ("fixed", 2)]
    long_lived = [1, 3, 4, 6]
    params = [params_of(bb, kind, 100 + m) for m, (kind, _) in enumerate(initial)]
    motions = [motion(bb, m) for m in range(len(initial))]
    batch = bb.AmclBatch(motions, params, adaptive=True, selective=True)
    mirror = bb.AmclBatch([motions[m] for m in long_lived], [params[m] for m in long_lived], adaptive=True, selective=True)
    ids, mirror_ids = maps.add(bb, batch), maps.add(bb, mirror)
    twins, which = {}, {}  # by slot

    def join(m, twin_motion, p, map_index):
        twins[m] = bb.Amcl(twin_motion, p)
        which[m] = map_index
        maps.assign(batch, ids, m, twins[m], map_index)
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        batch.initialize(m, mean, scene.initial_cov)
        twins[m].initialize(mean, scene.initial_cov)

    for m, (_, map_index) in enumerate(initial):
        join(m, motions[m], params[m], map_index)
    for j, m in enumerate(long_lived):
        mirror.update_map(j, mirror_ids[which[m]])
        mirror.initialize(j, scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m]), scene.initial_cov)

    def churn(t):
        """The membership changes before step t: (expected launches, call) pairs run in order."""
        if t == 3:  # slot 2 kept its particles in the step before: it leaves from the middle
            assert batch.member_size(2) == 1500
            n, _ = launches(batch, lambda: batch.remove_member(2))
            assert n == 1
            del twins[2]
            # the kept members' CDFs are current: pose samples of one of them take one launch right after the change
            n, samples = launches(batch, lambda: batch.sample_states([0, 0, 0, 0, 300, 0, 0, 0], 0xFFFFFFF0, present=[0, 0, 0, 0, 1, 0, 0, 0]))
            assert n == 1 and samples[4].tobytes() == twins[4].filter.sample_states(300, 0xFFFFFFF0).tobytes()
        if t == 4:  # the first and the last slot leave
            for m in (0, 7):
                batch.remove_member(m)
                del twins[m]
            assert [batch.member_active(m) for m in range(8)] == [False, True, False, True, True, True, True, False]
        if t == 5:  # a 32 768-particle member that records ancestors, in a batch where nobody did, takes the lowest slot
            p = bb.AmclParams(min_particles=32768, max_particles=32768, seed=700, resample_scheme=1, record_ancestors=True)
            assert batch.add_member(motion(bb, 0), p) == 0
            join(0, motion(bb, 0), p, 0)
            # into the vacated slot 2, then the vacated last slot, then a new slot 8
            for slot, (kind, map_index, extra) in zip((2, 7, 8), (("selective", 1, dict(record_ancestors=True)), ("kld", 2, {}),
                                                                  ("keep", 0, dict(record_ancestors=True)))):
                p = params_of(bb, kind, 700 + slot, **extra)
                assert batch.add_member(motion(bb, slot + 1), p) == slot
                join(slot, motion(bb, slot + 1), p, map_index)
            assert len(batch) == 9
        if t == 8:  # the big member leaves, and a fixed one takes its slot
            batch.remove_member(0)
            del twins[0]
            p = params_of(bb, "fixed", 800, record_ancestors=True)
            assert batch.add_member(motion(bb, 2), p) == 0
            join(0, motion(bb, 2), p, 2)

    for t in range(12):
        churn(t)
        k = len(batch)
        present = [m in twins and (t + m) % 5 != 4 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        meas = [measurement(bb, scene, t, m) if m in twins else None for m in range(k)]
        clustered = t % 3 == 2
        if clustered:
            got, est = batch.update_clustered(poses, meas, present)
        else:
            got = batch.update_measurements(poses, meas, present)
        for m in range(k):
            if not present[m]:
                assert got[m].updated == 0, (t, m)
                continue
            exp = feed_twin(bb, twins[m], poses[m], meas[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            if clustered and exp.updated:
                tm, tc = twins[m].filter.cluster_estimate()
                assert est[m][0].tobytes() == tm.tobytes() and est[m][1].tobytes() == tc.tobytes(), (t, m)
        # the unchanged batch of the long-lived members
        m_present = [present[m] for m in long_lived]
        m_meas = [meas[m] for m in long_lived]
        m_poses = [poses[m] for m in long_lived]
        if clustered:
            m_got, m_est = mirror.update_clustered(m_poses, m_meas, m_present)
        else:
            m_got = mirror.update_measurements(m_poses, m_meas, m_present)
        for j, m in enumerate(long_lived):
            assert result_bytes(m_got[j]) == result_bytes(got[m]), (t, m)
            assert mirror.particles(j)[0].tobytes() == batch.particles(m)[0].tobytes(), (t, m)
            assert mirror.particles(j)[1].tobytes() == batch.particles(m)[1].tobytes(), (t, m)
            if clustered and got[m].updated:
                assert m_est[j][0].tobytes() == est[m][0].tobytes(), (t, m)
        if t in (2, 6, 9, 11):
            assert_published_equal(bb, batch, twins, 0xFFFFFF00 + t)
    assert sorted(twins) == [0, 1, 2, 3, 4, 5, 6, 7, 8]


def test_remove_after_kept_step_and_published_after_resampled_step(bb, scene):
    """A selective member whose step kept its particles leaves; the other keeps a current CDF across the change (1 launch
    for its pose samples) until a resampling step, after which a change is followed by a rebuild (4 launches)."""
    p = [bb.AmclParams(min_particles=2000, max_particles=2000, seed=5 + m, selective_resampling=True, record_ancestors=True) for m in range(3)]
    motions = [motion(bb, m) for m in range(3)]
    batch = bb.AmclBatch(motions, p, selective=True)
    twins = {m: bb.Amcl(motions[m], p[m]) for m in range(3)}
    maps = Maps(bb, scene)
    ids = maps.add(bb, batch)
    for m in range(3):
        maps.assign(batch, ids, m, twins[m], 0)
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
        twins[m].initialize(scene.initial_mean, scene.initial_cov)
    seen = set()
    for t in range(10):
        k = len(batch)
        poses = [odometry(scene, t, m) for m in range(k)]
        pts = [scene.scans[t] if m in twins else None for m in range(k)]
        got = batch.update(poses, pts)
        kept = {}
        for m in twins:
            exp = twins[m].update(poses[m], pts[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            kept[m] = exp.updated and not exp.resampled
        # a membership change after every step: the member in slot 2 leaves and comes back as a new member
        if 2 in twins:
            batch.remove_member(2)
            del twins[2]
        else:
            q = bb.AmclParams(min_particles=2000, max_particles=2000, seed=50 + t, selective_resampling=True, record_ancestors=True)
            assert batch.add_member(motions[2], q) == 2
            twins[2] = bb.Amcl(motions[2], q)
            maps.assign(batch, ids, 2, twins[2], 0)
            batch.initialize(2, scene.initial_mean, scene.initial_cov)
            twins[2].initialize(scene.initial_mean, scene.initial_cov)
        for m in (0, 1):
            if not got[m].updated:
                continue
            n, s = launches(batch, lambda: batch.sample_states([500 if j == m else 0 for j in range(len(batch))], 0xFFFFFE00 + t,
                                                                 present=[j == m for j in range(len(batch))]))
            assert s[m].tobytes() == twins[m].filter.sample_states(500, 0xFFFFFE00 + t).tobytes(), (t, m)
            assert n == (1 if kept[m] else 4), (t, m, n)
            seen.add(kept[m])
        assert_published_equal(bb, batch, twins, 0xFFFFFD00 + t)
    assert seen == {True, False}


@pytest.mark.parametrize("k", [1, 16, 256])
def test_launch_counts(bb, scene, k):
    """A change takes 1 launch when some other member holds particles and 0 otherwise; a step, a clustered step, a pose
    draw and a histogram after churn take what they take on a freshly created batch of the same members."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    lfm = bb.LikelihoodFieldModelParam(**LFM)

    def member(m):
        return bb.AmclParams(min_particles=1000 if m % 4 == 1 else 2000, max_particles=2000, seed=m, resample_scheme=m % 2,
                             selective_resampling=m % 4 == 2, resample_interval=1 + m % 3)

    motions = [bb.DifferentialDriveModelParam() for _ in range(k)]
    empty = bb.AmclBatch(motions, [member(m) for m in range(k)], adaptive=True, selective=True)
    n, slot = launches(empty, lambda: empty.add_member(bb.StationaryModelParam(), member(k)))
    assert slot == k and n == 0
    assert launches(empty, lambda: empty.remove_member(0))[0] == 0

    churned = bb.AmclBatch(motions, [member(m) for m in range(k)], adaptive=True, selective=True)
    churned.set_likelihood_field_map(lfm, grid)
    map_id = churned.member_map(0)
    for m in range(k):
        churned.initialize(m, scene.initial_mean, scene.initial_cov)
    n, slot = launches(churned, lambda: churned.add_member(bb.DifferentialDriveModelParam(), member(k)))
    assert slot == k and n == 1
    # the only other member, with K = 1, is the new one, which holds no particles yet
    assert launches(churned, lambda: churned.remove_member(0))[0] == (1 if k > 1 else 0)
    churned.update_map(k, map_id)
    churned.initialize(k, scene.initial_mean, scene.initial_cov)
    fresh = bb.AmclBatch(motions[1:] + [bb.DifferentialDriveModelParam()], [member(m) for m in range(1, k + 1)], adaptive=True, selective=True)
    fresh.set_likelihood_field_map(lfm, grid)
    for m in range(k):
        fresh.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(3):
        pose = bb.se2(*scene.poses[t])
        a, r_churned = launches(churned, lambda: churned.update([pose] * (k + 1), [None] + [scene.scans[t]] * k))
        b, r_fresh = launches(fresh, lambda: fresh.update([pose] * k, [scene.scans[t]] * k))
        assert a == b and r_churned[0].updated == 0, (t, a, b)
        assert [result_bytes(r) for r in r_churned[1:]] == [result_bytes(r) for r in r_fresh], t
        a, (r_churned, _) = launches(churned, lambda: churned.update_clustered([pose] * (k + 1), [None] + [scene.scans[t + 3]] * k))
        b, (r_fresh, _) = launches(fresh, lambda: fresh.update_clustered([pose] * k, [scene.scans[t + 3]] * k))
        assert a == b, (t, a, b)
        a = launches(churned, lambda: churned.sample_states(100, t))[0]
        b = launches(fresh, lambda: fresh.sample_states(100, t))[0]
        assert a == b, (t, a, b)
        a = launches(churned, lambda: churned.particle_histograms())[0]
        b = launches(fresh, lambda: fresh.particle_histograms())[0]
        assert a == b, (t, a, b)


def build_three(bb, scene):
    maps = Maps(bb, scene)
    p = [bb.AmclParams(min_particles=1000, max_particles=1000, seed=60 + m, record_ancestors=True) for m in range(3)]
    batch = bb.AmclBatch([motion(bb, m) for m in range(3)], p)
    batch.set_likelihood_field_map(maps.lfm, maps.grid)
    for m in range(3):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(2):
        batch.update([odometry(scene, t, m) for m in range(3)], [scene.scans[t]] * 3)
    batch.remove_member(1)
    return batch


def test_vacant_slot_rules(bb, scene):
    batch, clean = build_three(bb, scene), build_three(bb, scene)
    assert len(batch) == 3 and [batch.member_active(m) for m in range(3)] == [True, False, True]
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.member_active(3)
    assert e.value.status == INVALID
    t = 2
    poses = [odometry(scene, t, m) for m in range(3)]
    pts = [scene.scans[t], None, scene.scans[t]]
    vacant = [1, 1, 1]
    refused = [
        lambda: batch.update(poses, pts, present=vacant),
        lambda: batch.update_measurements(poses, pts, present=vacant),
        lambda: batch.update_clustered(poses, pts, present=vacant),
        lambda: batch.cluster_estimates(present=vacant),
        lambda: batch.particle_histograms(present=vacant),
        lambda: batch.sample_states([10, 10, 10], 0, present=vacant),
        lambda: batch.initialize(1, scene.initial_mean, scene.initial_cov),
        lambda: batch.initialize_from_map(1),
        lambda: batch.initialize_states(1, np.array([[1.0, 0.0, 1.0, 1.0]])),
        lambda: batch.force_update(1),
        lambda: batch.particles(1),
        lambda: batch.ancestors(1),
        lambda: batch.member_size(1),
        lambda: batch.update_map(1, 0),
        lambda: batch.member_map(1),
        lambda: batch.cluster_estimate(1),
        lambda: batch.remove_member(1),
    ]
    before = batch.launch_count()
    for i, call in enumerate(refused):
        with pytest.raises(bb.BelugaB200Error) as e:
            call()
        assert e.value.status == INVALID, i
        assert "vacant" in str(e.value), i
    assert batch.launch_count() == before
    # present == None skips the vacant slot; the refused calls changed nothing
    for t in range(2, 6):
        poses = [odometry(scene, t, m) for m in range(3)]
        pts = [scene.scans[t], None, scene.scans[t]]
        for m in (0, 2):
            batch.force_update(m)
            clean.force_update(m)
        a, b = batch.update(poses, pts), clean.update(poses, pts)
        assert a[1].updated == 0 and a[0].updated == 1 and a[2].updated == 1
        assert [result_bytes(r) for r in a] == [result_bytes(r) for r in b], t
        for m in (0, 2):
            assert batch.particles(m)[0].tobytes() == clean.particles(m)[0].tobytes(), (t, m)
            assert batch.ancestors(m).tobytes() == clean.ancestors(m).tobytes(), (t, m)
    # the last member cannot leave
    batch.remove_member(2)
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.remove_member(0)
    assert e.value.status == STATE and batch.member_active(0)


def test_new_member_inherits_nothing(bb, scene):
    """A member added to a slot whose earlier occupant had a map, particles, ancestors, a current CDF and a scan table starts
    as a member of a freshly created batch does."""
    batch = build_three(bb, scene)
    batch.remove_member(2)  # it resampled: ancestors; slot 1 is vacant already
    q = bb.AmclParams(min_particles=1000, max_particles=1000, seed=99, record_ancestors=True)
    assert batch.add_member(motion(bb, 0), q) == 1
    assert batch.member_map(1) == -1 and batch.member_size(1) == 0
    assert not np.any(batch.ancestors(1))
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.cluster_estimates(present=[0, 1, 0])
    assert e.value.status == STATE  # no particles
    batch.initialize(1, scene.initial_mean, scene.initial_cov)
    poses = [odometry(scene, 3, m) for m in range(3)]
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.update(poses, [None, scene.scans[3], None], present=[0, 1, 0])
    assert e.value.status == STATE and "no map" in str(e.value)
    assert not np.any(batch.ancestors(1))
    # its CDF is rebuilt for its first pose samples: 4 launches
    assert launches(batch, lambda: batch.sample_states([0, 10, 0], 0, present=[0, 1, 0]))[0] == 4
    twin = bb.Amcl(motion(bb, 0), q)
    twin.initialize(scene.initial_mean, scene.initial_cov)
    batch.update_map(1, batch.member_map(0))
    twin.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    for t in range(3, 7):
        poses = [odometry(scene, t, m) for m in range(3)]
        got = batch.update(poses, [scene.scans[t], scene.scans[t], None])
        exp = twin.update(poses[1], scene.scans[t])
        assert_member_equals_twin(batch, 1, twin, got[1], exp, t)


@pytest.mark.parametrize("flags,bad,needle", [
    (0, dict(min_particles=500), "fixed particle count"),
    (1, dict(selective_resampling=True), "selective"),
    (3, dict(device=1), "one device"),
    (3, dict(max_particles=32769), "max_particles"),
])
def test_add_member_validation(bb, scene, flags, bad, needle):
    import ctypes as C

    from beluga_b200 import _capi

    base = [bb.AmclParams(min_particles=1000, max_particles=1000, seed=m) for m in range(3)]
    motions = [motion(bb, m) for m in range(3)]
    batch = bb.AmclBatch(motions, base, adaptive=bool(flags & 1), selective=bool(flags & 2))
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    for m in range(3):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    kw = dict(min_particles=1000, max_particles=1000, seed=9)
    kw.update(bad)
    wrong = bb.AmclParams(**kw)
    # what create says of the same member in the same position
    lib = _capi.load()
    p = (_capi.AmclParam * 4)(*[q.c() for q in base + [wrong]])
    mo = (_capi.MotionParam * 4)(*[q.c_motion() for q in motions + [motion(bb, 3)]])
    h = C.c_void_p()
    assert lib.bb200_amcl_batch_create_with_flags(p, mo, 4, flags, C.byref(h)) == INVALID and not h
    expected = lib.bb200_create_error().decode()
    assert needle in expected and "member 3" in expected
    before = (batch.launch_count(), [batch.particles(m)[0].tobytes() for m in range(3)])
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.add_member(motion(bb, 3), wrong)
    assert e.value.status == INVALID and str(e.value).endswith(expected)
    assert len(batch) == 3 and len(batch.params) == 3
    assert (batch.launch_count(), [batch.particles(m)[0].tobytes() for m in range(3)]) == before
