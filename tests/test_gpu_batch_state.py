"""State blobs on the GPU: a filter's complete state exported from a batch or a standalone Amcl and restored into a fresh
batch (create_from_states), a running batch (import_member) or a standalone Amcl (create_from_state) continues byte for
byte as the filter that never moved: update results, particles, weights and ancestors after every step, update_clustered
estimates, cluster estimates, histograms, and pose samples drawn right after the restore (the current-CDF path).  Also
covered: standalone to batch, a round trip through a file, launch counts, refusals and rollback."""
import ctypes as C
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
INVALID, STATE, CAPACITY = -1, -4, -5


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


def feed_solo(bb, solo, pose, meas):
    if isinstance(meas, bb.LaserScan):
        return solo.update_scan(pose, meas.ranges, meas.angle_min, meas.angle_increment, meas.min_range, meas.max_range, meas.max_beams,
                                meas.laser_origin)
    if isinstance(meas, bb.PointCloud):
        return solo.update_point_cloud(pose, meas.data, meas.point_step, meas.x_offset, meas.dtype, meas.origin, meas.n_points)
    return solo.update(pose, meas)


def solo_histogram(bb, solo, linear, angular):
    from beluga_b200 import _capi

    f = solo.filter
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, None, 0, C.byref(n), C.byref(top)) == 0
    bins = np.empty(max(n.value, 1), dtype=bb._CELL_DTYPE)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, bins.ctypes.data_as(C.POINTER(_capi.ClusterCell)), n.value,
                                                  C.byref(n), C.byref(top)) == 0
    return bins[:n.value], top.value


class Maps:
    """Likelihood field, prob likelihood field and beam model on one grid: the same three maps in every batch."""

    def __init__(self, bb, scene):
        self.grid = bb.OccupancyGrid(scene.cells, scene.resolution)
        self.lfm = bb.LikelihoodFieldModelParam(**LFM)
        self.beam = bb.BeamModelParam(sigma_hit=0.2, lambda_short=0.1, beam_max_range=20.0)
        self.kinds = [(bb.SENSOR_LIKELIHOOD_FIELD, self.lfm), (bb.SENSOR_LIKELIHOOD_FIELD_PROB, self.lfm), (bb.SENSOR_BEAM, self.beam)]

    def add(self, batch):
        return [batch.add_likelihood_field_map(self.lfm, self.grid), batch.add_likelihood_field_map(self.lfm, self.grid, prob=True),
                batch.add_beam_map(self.beam, self.grid)]

    def attach(self, solo, which):
        sensor, params = self.kinds[which]
        solo.update_map(sensor, params, self.grid)


def params_of(bb, kind, seed, **extra):
    """fixed: 2000 particles; kld: 500..2000; selective: 2000, selective resampling; keep: 1500 that never resample."""
    table = dict(fixed=dict(min_particles=2000, max_particles=2000), kld=dict(min_particles=500, max_particles=2000),
                 selective=dict(min_particles=2000, max_particles=2000, selective_resampling=True),
                 keep=dict(min_particles=1500, max_particles=1500, resample_interval=1000))
    return bb.AmclParams(seed=seed, resample_scheme=seed % 2, **table[kind], **extra)


class Copy:
    """Where one filter lives: a batch slot or a standalone Amcl."""

    def __init__(self, owner, slot=None):
        self.owner, self.slot = owner, slot

    def particles(self):
        if self.slot is None:
            return self.owner.particles()
        st, w = self.owner.particles(self.slot)
        n = self.owner.member_size(self.slot)
        return st[:n], w[:n]

    def ancestors(self):
        return self.owner.filter.ancestors() if self.slot is None else self.owner.ancestors(self.slot)[:self.owner.member_size(self.slot)]


def step_batch(batch, slots, poses, meas, present, clustered):
    """One step of `batch` in which filter m (at slots[m]) gets poses[m] and meas[m]; the batch's other occupied slots
    (owned by the caller) are absent.  Returns per filter (result, clustered estimate or None)."""
    k = len(batch)
    b_poses = [np.array([1.0, 0.0, 0.0, 0.0])] * k
    b_meas, b_present = [None] * k, [False] * k
    for m, s in slots.items():
        b_poses[s], b_meas[s], b_present[s] = poses[m], meas[m], present[m]
    if clustered:
        got, est = batch.update_clustered(b_poses, b_meas, b_present)
    else:
        got, est = batch.update_measurements(b_poses, b_meas, b_present), [None] * k
    return {m: (got[s], est[s]) for m, s in slots.items()}


def assert_same(twin, copy, got, exp, where):
    assert result_bytes(got) == result_bytes(exp), where
    ts, tw = twin.particles()
    gs, gw = copy.particles()
    assert gs.tobytes() == ts.tobytes() and gw.tobytes() == tw.tobytes(), where
    if twin.params.record_ancestors:
        assert copy.ancestors().tobytes() == twin.filter.ancestors().tobytes(), where


def test_restored_copies_continue_as_their_twins(bb, scene):
    maps = Maps(bb, scene)
    kinds = [("fixed", 0), ("kld", 1), ("keep", 2), ("selective", 0), ("keep", 1), ("kld", 2), ("selective", 1), ("fixed", 2)]
    k = len(kinds)
    params = [params_of(bb, kind, 100 + m, record_ancestors=(m == 0)) for m, (kind, _) in enumerate(kinds)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params, adaptive=True, selective=True)
    ids = maps.add(batch)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    for m, (_, which) in enumerate(kinds):
        batch.update_map(m, ids[which])
        maps.attach(twins[m], which)
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        batch.initialize(m, mean, scene.initial_cov)
        twins[m].initialize(mean, scene.initial_cov)
    # A second running batch with members of its own, one of them removed: restored members fill the vacant slot first.
    own_params = [params_of(bb, kind, 900 + j) for j, kind in enumerate(("fixed", "selective", "kld"))]
    own_motions = [motion(bb, j + 1) for j in range(3)]
    host = bb.AmclBatch(own_motions, own_params, adaptive=True, selective=True)
    host_ids = maps.add(host)
    own = {j: bb.Amcl(own_motions[j], own_params[j]) for j in range(3)}
    for j in range(3):
        host.update_map(j, host_ids[j])
        maps.attach(own[j], j)
        host.initialize(j, scene.initial_mean, scene.initial_cov)
        own[j].initialize(scene.initial_mean, scene.initial_cov)
    host.remove_member(1)
    del own[1]

    copies = {m: [Copy(batch, m)] for m in range(k)}  # every place each filter lives, compared with its twin after every step
    batches = {id(batch): batch}

    def restore(blobs, tag):
        # (a) a fresh batch
        fresh = bb.AmclBatch.from_states(blobs, adaptive=True, selective=True)
        fresh_ids = maps.add(fresh)
        for m, (_, which) in enumerate(kinds):
            fresh.update_map(m, fresh_ids[which])
            copies[m].append(Copy(fresh, m))
        batches[id(fresh)] = fresh
        # (b) the running batch: the vacant slot, then appended slots
        for m, (_, which) in enumerate(kinds):
            slot = host.import_member(blobs[m], host_ids[which])
            assert slot == ((1 if m == 0 else m + 2) if tag == "first" else k + 2 + m), (tag, m, slot)
            copies[m].append(Copy(host, slot))
        # (c) standalone filters
        for m, (_, which) in enumerate(kinds):
            solo = bb.Amcl.from_state(blobs[m])
            maps.attach(solo, which)
            copies[m].append(Copy(solo))
        # pose samples right after the restore: current CDFs draw in one launch, stale ones are rebuilt
        draws = {m: twins[m].filter.sample_states(400, 0xFFFFFFF0) for m in range(k)}
        for b in (fresh, host):
            counts = [0] * len(b)
            slots = {m: next(c.slot for c in copies[m][-3:] if c.owner is b) for m in range(k)}
            for m, s in slots.items():
                counts[s] = 400
            n, got = launches(b, lambda: b.sample_states(counts, 0xFFFFFFF0, present=[c > 0 for c in counts]))
            stale = any(blob_cdf_stale(blobs[m]) for m in range(k))
            assert n == (4 if stale else 1), (tag, n)
            for m, s in slots.items():
                assert got[s].tobytes() == draws[m].tobytes(), (tag, m)
        for m in range(k):
            assert copies[m][-1].owner.filter.sample_states(400, 0xFFFFFFF0).tobytes() == draws[m].tobytes(), (tag, m)

    kept_seen = resampled_seen = 0
    for t in range(11):
        if t in (3, 7):
            # t = 3: after a step in which the keep and (mostly) selective members kept their particles; t = 7: after one
            # in which every member was present and the fixed and KLD ones resampled
            source = batch if t == 3 else copies[0][1].owner  # the second checkpoint is taken from the restored fresh batch
            slots = [c.slot for m in range(k) for c in copies[m] if c.owner is source]
            n, blobs = launches(source, lambda: source.export_members())
            assert n == 1, n
            blobs = [blobs[s] for s in slots]
            for m in range(k):
                assert blobs[m] == twins[m].export_state(), (t, m)  # a member's blob is its twin's, byte for byte
            kept_seen += sum(not blob_cdf_stale(b) for b in blobs)
            resampled_seen += sum(blob_cdf_stale(b) for b in blobs)
            restore(blobs, "first" if t == 3 else "second")
        present = [t == 6 or (t + m) % 5 != 4 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        meas = [measurement(bb, scene, t, m) for m in range(k)]
        clustered = t % 3 == 2
        exp = [feed_solo(bb, twins[m], poses[m], meas[m]) if present[m] else None for m in range(k)]
        # the host's own members step alongside
        own_poses = {j: odometry(scene, t, 10 + j) for j in own}
        own_meas = {j: measurement(bb, scene, t, j) for j in own}
        for b in batches.values():
            slots = {m: c.slot for m in range(k) for c in copies[m] if c.owner is b}
            got = step_batch(b, slots, poses, meas, present, clustered)
            for m, (r, est) in got.items():
                if not present[m]:
                    assert r.updated == 0
                    continue
                assert_same(twins[m], Copy(b, slots[m]), r, exp[m], (t, m))
                if clustered and exp[m].updated:
                    tm, tc = twins[m].filter.cluster_estimate()
                    assert est[0].tobytes() == tm.tobytes() and est[1].tobytes() == tc.tobytes(), (t, m)
        host_slots = {m: c.slot for m in range(k) for c in copies[m] if c.owner is host}
        k_host = len(host)
        h_poses = [np.array([1.0, 0.0, 0.0, 0.0])] * k_host
        h_meas, h_present = [None] * k_host, [False] * k_host
        for m, s in host_slots.items():
            h_poses[s], h_meas[s], h_present[s] = poses[m], meas[m], present[m]
        for j in own:
            h_poses[j], h_meas[j], h_present[j] = own_poses[j], own_meas[j], True
        got = host.update_measurements(h_poses, h_meas, h_present)
        for j in own:
            assert_same(own[j], Copy(host, j), got[j], feed_solo(bb, own[j], own_poses[j], own_meas[j]), (t, "own", j))
        for m, s in host_slots.items():
            if present[m]:
                assert_same(twins[m], Copy(host, s), got[s], exp[m], (t, "host", m))
        for m in range(k):
            for c in copies[m]:
                if c.slot is None and present[m]:
                    assert_same(twins[m], c, feed_solo(bb, c.owner, poses[m], meas[m]), exp[m], (t, "solo", m))
        if t in (4, 8, 10):
            for b in list(batches.values()) + [host]:
                slots = {m: c.slot for m in range(k) for c in copies[m] if c.owner is b}
                est = b.cluster_estimates(present=[s in slots.values() for s in range(len(b))])
                hists = b.particle_histograms([s in slots.values() for s in range(len(b))], 0.05, 0.05)
                for m, s in slots.items():
                    tm, tc = twins[m].filter.cluster_estimate()
                    assert est[s][0].tobytes() == tm.tobytes() and est[s][1].tobytes() == tc.tobytes(), (t, m)
                    bins, top = solo_histogram(bb, twins[m], 0.05, 0.05)
                    assert hists[s][0].tobytes() == bins.tobytes() and np.float64(hists[s][1]) == np.float64(top), (t, m)
    assert kept_seen > 0 and resampled_seen > 0, (kept_seen, resampled_seen)
    assert len(host) == 3 + 2 * k - 1


def blob_cdf_stale(blob):
    """Whether a blob's CDF is stale: the cdf_current flag of its particle-set section (DESIGN.md, state blobs)."""
    sections = struct.unpack_from("<8Q", blob, 24)
    set_offset = 88 + sum(sections[:3])
    return struct.unpack_from("<I", blob, set_offset + 40)[0] == 0


def test_standalone_to_batch_and_through_a_file(bb, scene, tmp_path):
    maps = Maps(bb, scene)
    params = [params_of(bb, "kld", 40, record_ancestors=True), params_of(bb, "selective", 41)]
    motions = [motion(bb, 0), motion(bb, 1)]
    solos = [bb.Amcl(motions[m], params[m]) for m in range(2)]
    twins = [bb.Amcl(motions[m], params[m]) for m in range(2)]
    for m in range(2):
        for f in (solos[m], twins[m]):
            maps.attach(f, m)
            f.initialize(scene.initial_mean, scene.initial_cov)
    for t in range(3):
        for m in range(2):
            pose, meas = odometry(scene, t, m), measurement(bb, scene, t, m)
            assert result_bytes(feed_solo(bb, solos[m], pose, meas)) == result_bytes(feed_solo(bb, twins[m], pose, meas))
    blobs = [s.export_state() for s in solos]
    path = tmp_path / "robot1.state"
    path.write_bytes(blobs[1])
    batch = bb.AmclBatch([motion(bb, 2)], [params_of(bb, "fixed", 50)], adaptive=True, selective=True)
    ids = maps.add(batch)
    slots = [batch.import_member(blobs[0], ids[0])]
    replay = bb.Amcl.from_state(path.read_bytes())
    maps.attach(replay, 1)
    for t in range(3, 9):
        pose, meas = odometry(scene, t, 0), measurement(bb, scene, t, 0)
        got = step_batch(batch, {0: slots[0]}, [pose], [meas], [True], False)[0][0]
        assert_same(twins[0], Copy(batch, slots[0]), got, feed_solo(bb, twins[0], pose, meas), (t, 0))
        pose, meas = odometry(scene, t, 1), measurement(bb, scene, t, 1)
        assert_same(twins[1], Copy(replay), feed_solo(bb, replay, pose, meas), feed_solo(bb, twins[1], pose, meas), (t, 1))


@pytest.mark.parametrize("k", [1, 16, 256])
def test_launch_counts(bb, scene, k):
    params = [bb.AmclParams(min_particles=2000, max_particles=2000, seed=m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    for m in range(k):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    n, blobs = launches(batch, lambda: batch.export_members())
    assert n == 1
    restored = bb.AmclBatch.from_states(blobs)
    assert restored.launch_count() == 1
    assert [restored.export_member(m) for m in range(k)] == blobs
    n_add, _ = launches(batch, lambda: batch.add_member(motion(bb, 0), bb.AmclParams(min_particles=2000, max_particles=2000, seed=7)))
    n_import, _ = launches(batch, lambda: batch.import_member(blobs[0]))
    assert n_add == 1 and n_import == 2


def test_refusals_leave_the_batch_unchanged(bb, scene):
    from beluga_b200 import _capi

    params = [bb.AmclParams(min_particles=1000, max_particles=1000, seed=m, record_ancestors=(m == 1)) for m in range(3)]
    batch = bb.AmclBatch([motion(bb, m) for m in range(3)], params)
    for m in range(3):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    batch.remove_member(2)
    before = batch.export_members()
    assert before[2] is None
    good = before[0]

    def refused(blob, status):
        with pytest.raises(bb.BelugaB200Error) as e:
            batch.import_member(blob)
        assert e.value.status == status, e.value
        assert len(batch) == 3 and not batch.member_active(2)
        assert batch.export_members() == before
        return str(e.value)

    assert "truncated" in refused(good[:40], INVALID)
    assert "header gives" in refused(good[:-8], INVALID)
    assert "magic" in refused(b"X" + good[1:], INVALID)
    assert "version 2" in refused(good[:8] + struct.pack("<I", 2) + good[12:], INVALID)
    corrupt = bytearray(good)
    struct.pack_into("<Q", corrupt, 24 + 8 * 4, 32 * 999)  # the states section's length
    assert "states" in refused(bytes(corrupt), INVALID)
    kld = bb.Amcl(motion(bb, 0), bb.AmclParams(min_particles=100, max_particles=1000))
    assert "fixed particle count" in refused(kld.export_state(), INVALID)
    big = bb.Amcl(motion(bb, 0), bb.AmclParams(min_particles=40000, max_particles=40000))
    big.initialize(scene.initial_mean, scene.initial_cov)
    assert "32768" in refused(big.export_state(), INVALID)
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.export_member(2)
    assert e.value.status == INVALID
    with pytest.raises(bb.BelugaB200Error) as e:
        batch.export_members([1, 0, 1])
    assert e.value.status == INVALID
    lib = _capi.load()
    size = C.c_uint64(0)
    buf = C.create_string_buffer(10)
    assert lib.bb200_amcl_batch_export_member(batch._h, 0, buf, 10, C.byref(size)) == CAPACITY and size.value == len(good)
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.Amcl.from_state(good[:-1])
    assert e.value.status == INVALID
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch.from_states([good, b"nope" * 30])
    assert e.value.status == INVALID and "member 1" in str(e.value)
    assert batch.export_members() == before
    # a restored filter without a map cannot update, as a new one cannot
    solo = bb.Amcl.from_state(good)
    with pytest.raises(bb.BelugaB200Error) as e:
        solo.update(odometry(scene, 0, 0), scene.scans[0])
    assert e.value.status == STATE
    # sharded filters have no state blob
    sharded = bb.ShardedAmcl(motion(bb, 0), bb.AmclParams(min_particles=2000, max_particles=2000), [0, 0])
    shard = lib.bb200_sharded_amcl_shard(sharded._h, 0)
    assert lib.bb200_amcl_export_state(shard, None, 0, C.byref(size)) == STATE
