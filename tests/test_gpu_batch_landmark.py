"""The landmark and bearing sensor models in a batch on the GPU: every member on a landmark map equals a standalone Amcl
with the same parameters, seed and detections (driven by Amcl.update_landmarks), byte for byte -- update results,
particles, weights, ancestors and the cluster estimate -- under both models, both resampling schemes, fixed, KLD and
selective batches, one landmark map (its views in the parameter block) and several (the batch's map table), recovery
injection from the box, initialize_from_map, detection and candidate counts past the kernel's shared-memory chunks (32
detections, 256 candidates), zero detections and categories the map lacks.  Also: a mixed step with every other sensor
form and its launch count, update_clustered, grid <-> landmark map moves and state blobs, membership changes, the oracle's
factors and every refusal."""
import math
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _landmark_oracle as lo  # noqa: E402

pytestmark = pytest.mark.gpu

STATE, INVALID = -4, -1
MOTION = (0.1, 0.05, 0.1, 0.05)
SENSOR_POSE = (0.0, 0.0, 1.0, 0.2, -1.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.5)  # a camera looking along the robot's x
SIGMA = (0.5, 0.3, 1e-3)


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


def random_map(rng, n, n_categories, extent=6.0):
    pos = np.stack([rng.uniform(-extent, extent, n), rng.uniform(-extent, extent, n), rng.uniform(0.0, 2.0, n)], axis=1)
    return pos, rng.integers(0, n_categories, n).astype(np.uint32)


def random_detections(rng, n, n_categories, absent=False):
    """n detections of the map's categories; with `absent`, categories up to n_categories, one the map lacks."""
    pos = np.stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(0.0, 2.0, n)], axis=1)
    return pos, rng.integers(0, n_categories + (1 if absent else 0), n).astype(np.uint32)


def sensor(bb, model):
    return bb.SENSOR_LANDMARK if model == "landmark" else bb.SENSOR_BEARING


def model_param(bb, model):
    return bb.LandmarkModelParam(*SIGMA) if model == "landmark" else bb.BearingModelParam(SIGMA[1], SENSOR_POSE)


def add_map(bb, batch, model, lmap):
    return batch.add_landmark_map(model_param(bb, model), lmap) if model == "landmark" else batch.add_bearing_map(model_param(bb, model), lmap)


def odometry(t, m):
    th = 0.1 * (t + 1) + 0.01 * m
    if t % 5 == 4:  # the previous pose: below update_min_d, only a forced update runs
        th -= 0.1
        t -= 1
    return np.array([math.cos(th), math.sin(th), 0.3 * (t + 1) + 0.02 * m, 0.1 * t])


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


def assert_twin(batch, m, twin, got, exp, where):
    assert result_bytes(got) == result_bytes(exp), where
    gs, gw = batch.particles(m)
    ts, tw = twin.particles()
    n = len(ts)
    assert gs[:n].tobytes() == ts.tobytes() and gw[:n].tobytes() == tw.tobytes(), where
    if exp.updated and exp.resampled:
        assert np.array_equal(batch.ancestors(m)[:n], twin.filter.ancestors()[:n]), where


def assert_cluster_twin(batch, m, twin, where):
    gm, gc = batch.cluster_estimate(m)
    tm, tc = twin.filter.cluster_estimate()
    assert gm.tobytes() == tm.tobytes() and gc.tobytes() == tc.tobytes(), where


class Fleet:
    """A batch and one standalone twin per member, each member on one of `maps` ((model, LandmarkMap) pairs)."""

    def __init__(self, bb, params, maps, assign, adaptive=False, selective=False, from_map=False):
        self.bb = bb
        motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in params]
        self.batch = bb.AmclBatch(motions, params, adaptive=adaptive, selective=selective)
        ids = [add_map(bb, self.batch, model, lmap) for model, lmap in maps]
        self.twins = []
        for m, p in enumerate(params):
            model, lmap = maps[assign[m]]
            self.batch.update_map(m, ids[assign[m]])
            t = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), p)
            t.update_map(sensor(bb, model), model_param(bb, model), lmap)
            if from_map:
                self.batch.initialize_from_map(m)
                t.initialize_from_map()
            else:
                mean, cov = [0.5 + 0.1 * m, -0.5, 0.3], np.diag([0.5, 0.5, 0.2])
                self.batch.initialize(m, mean, cov)
                t.initialize(mean, cov)
            self.twins.append(t)

    def step(self, t, detections, present=None, clustered=False):
        k = len(self.twins)
        poses = np.stack([odometry(t, m) for m in range(k)])
        meas = [self.bb.Detections(*detections[m]) for m in range(k)]
        if clustered:
            got, est = self.batch.update_clustered(poses, meas, present)
        else:
            got, est = self.batch.update_measurements(poses, meas, present), None
        for m, twin in enumerate(self.twins):
            if present is not None and not present[m]:
                assert got[m].updated == 0
                continue
            exp = twin.update_landmarks(poses[m], *detections[m])
            assert_twin(self.batch, m, twin, got[m], exp, (t, m))
        return got, est


CASES = {
    "multinomial": dict(kw=dict(resample_scheme=0), flags={}),
    "systematic": dict(kw=dict(resample_scheme=1), flags={}),
    "kld": dict(kw=dict(kld=True), flags=dict(adaptive=True)),
    "selective": dict(kw=dict(selective_resampling=True, resample_scheme=1), flags=dict(selective=True)),
    "injection": dict(kw=dict(recovery_probability_override=0.05), flags={}),
}


def fleet_params(bb, case, sizes):
    c = dict(CASES[case]["kw"])
    kld = c.pop("kld", False)
    out = []
    for m, n in enumerate(sizes):
        lo_n = max(1, n // 4) if kld else n
        out.append(bb.AmclParams(update_min_d=0.05, update_min_a=0.05, min_particles=lo_n, max_particles=n, seed=300 + m, record_ancestors=True, **c))
    return out


@pytest.mark.parametrize("several_maps", [False, True], ids=["one_map", "several_maps"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_members_equal_standalone_twins(bb, case, several_maps):
    rng = np.random.default_rng(2 * sorted(CASES).index(case) + several_maps)
    # 600 landmarks in 2 categories: candidate slices past the 256-candidate chunk; 20 in 5 categories for the others
    big, small = random_map(rng, 600, 2), random_map(rng, 20, 5)
    maps = [("landmark", bb.LandmarkMap(*big)), ("bearing", bb.LandmarkMap(*small)), ("bearing", bb.LandmarkMap(*big)),
            ("landmark", bb.LandmarkMap(*small, [-7.0, -7.0, 0.0], [7.0, 7.0, 0.0]))]
    n_categories = [2, 5, 2, 5]
    sizes = (1, 255, 2000, 700)
    assign = [0, 1, 2, 3] if several_maps else [0, 0, 0, 0]
    if not several_maps and case in ("systematic", "injection"):
        maps, n_categories = maps[1:2], [5] * 4  # the single map is a bearing map in some cases
    f = Fleet(bb, fleet_params(bb, case, sizes), maps, assign, **CASES[case]["flags"])
    for t in range(8):
        counts = [(0, 1, 40, 3), (33, 0, 5, 2), (4, 64, 0, 1), (7, 2, 2, 0), (1, 5, 40, 33), (3, 3, 3, 3), (32, 4, 1, 0), (2, 2, 2, 2)][t]
        dets = [random_detections(rng, counts[m], n_categories[assign[m]] if several_maps else n_categories[0], absent=(t == 3)) for m in range(4)]
        f.step(t, dets, present=[1, 1, 0, 1] if t == 6 else None)
    for m, twin in enumerate(f.twins):
        assert_cluster_twin(f.batch, m, twin, m)


@pytest.mark.parametrize("model", ["landmark", "bearing"])
def test_initialize_from_map_draws_the_members_box(bb, model):
    rng = np.random.default_rng(3)
    pos, cat = random_map(rng, 40, 4)
    maps = [(model, bb.LandmarkMap(pos, cat)), (model, bb.LandmarkMap(pos, cat, [-2.0, -3.0, 0.0], [5.0, 1.0, 0.0]))]
    params = fleet_params(bb, "injection", (1500, 300, 64))
    f = Fleet(bb, params, maps, [0, 1, 0], from_map=True)
    for m, twin in enumerate(f.twins):
        gs, gw = f.batch.particles(m)
        ts, tw = twin.particles()
        assert gs.tobytes() == ts.tobytes() and gw.tobytes() == tw.tobytes(), m
    for t in range(4):
        f.step(t, [random_detections(rng, 6, 4) for _ in range(3)])


def test_update_clustered_equals_update_then_cluster_estimates(bb):
    rng = np.random.default_rng(9)
    big = random_map(rng, 100, 3)
    maps = [("landmark", bb.LandmarkMap(*big)), ("bearing", bb.LandmarkMap(*big))]
    params = fleet_params(bb, "multinomial", (500, 1200, 40))
    a = Fleet(bb, params, maps, [0, 1, 0])
    b = Fleet(bb, params, maps, [0, 1, 0])
    for t in range(5):
        dets = [random_detections(rng, 5 + m, 3) for m in range(3)]
        ra, est = a.step(t, dets, clustered=True)
        rb, _ = b.step(t, dets)
        want = b.batch.cluster_estimates(present=[r.updated for r in rb])
        for m in range(3):
            assert result_bytes(ra[m]) == result_bytes(rb[m])
            if rb[m].updated:
                assert est[m][0].tobytes() == want[m][0].tobytes() and est[m][1].tobytes() == want[m][1].tobytes(), (t, m)


def lfm_scene(bb):
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=120, n_beams=60, steps=6)


def test_mixed_step_launch_count_and_twins(bb):
    """Scans on a likelihood field, points on a beam map, landmark and bearing members and weighed members in one
    update_begin / _end: every member equals its twin, and the step launches 4 + 1 (scans) + 1 (field) + 1 or 2 (beam) + 1
    (landmark) + 1 (weigh), at 4 members as at 64."""
    pytest.importorskip("torch")

    sc = lfm_scene(bb)
    rng = np.random.default_rng(17)
    pos, cat = random_map(rng, 50, 4)
    lmap = bb.LandmarkMap(pos, cat)
    counts = []
    for k in (4, 64):
        # landmark and bearing members take one form: 4 members hold every form
        kinds = [("field", "landmark", "beam", "weighed", "bearing")[m % 5] for m in range(k)]
        params = [bb.AmclParams(update_min_d=0.0, update_min_a=0.0, min_particles=300 + 10 * m, max_particles=300 + 10 * m, seed=m,
                                record_ancestors=True) for m in range(k)]
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)], params)
        grid = bb.OccupancyGrid(sc.cells, sc.resolution)
        ids = {"field": batch.add_likelihood_field_map(bb.LikelihoodFieldModelParam(), grid), "beam": batch.add_beam_map(bb.BeamModelParam(), grid),
               "landmark": batch.add_landmark_map(model_param(bb, "landmark"), lmap), "bearing": batch.add_bearing_map(model_param(bb, "bearing"), lmap)}
        ids["weighed"] = ids["landmark"]
        twins = []
        for m in range(k):
            batch.update_map(m, ids[kinds[m]])
            t = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), params[m])
            if kinds[m] == "field":
                t.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(), grid)
            elif kinds[m] == "beam":
                t.update_map(bb.SENSOR_BEAM, bb.BeamModelParam(), grid)
            else:
                model = "bearing" if kinds[m] == "bearing" else "landmark"
                t.update_map(sensor(bb, model), model_param(bb, model), lmap)
            mean = sc.initial_mean + np.array([0.01 * m, 0.0, 0.0])
            batch.initialize(m, mean, sc.initial_cov)
            t.initialize(mean, sc.initial_cov)
            twins.append(t)
        for t_step in range(1, 4):
            x, y, th = sc.poses[t_step]
            poses = np.stack([np.array([math.cos(th), math.sin(th), x, y])] * k)
            dets = [random_detections(rng, 6, 4) for _ in range(k)]
            scan = bb.LaserScan(np.hypot(sc.scans[t_step][:, 0], sc.scans[t_step][:, 1]).astype(np.float32), -math.pi / 2, math.pi / (len(sc.scans[t_step]) - 1))
            meas = []
            for m in range(k):
                meas.append({"field": scan, "beam": sc.scans[t_step], "landmark": bb.Detections(*dets[m]), "bearing": bb.Detections(*dets[m]),
                             "weighed": None}[kinds[m]])

            def weigh(members, states, factors):
                for s, f in zip(states, factors):
                    f.copy_(toy_model(s))

            before = batch.launch_count()
            got = batch.update_weighted(poses, meas, weigh)
            counts.append(batch.launch_count() - before)
            for m in range(k):
                if kinds[m] == "field":
                    exp = twins[m].update_scan(poses[m], scan.ranges, scan.angle_min, scan.angle_increment)
                elif kinds[m] == "beam":
                    exp = twins[m].update(poses[m], sc.scans[t_step])
                elif kinds[m] == "weighed":
                    exp = twins[m].update_weighted(poses[m], lambda s, f: f.copy_(toy_model(s)))
                else:
                    exp = twins[m].update_landmarks(poses[m], *dets[m])
                assert_twin(batch, m, twins[m], got[m], exp, (k, t_step, m))
        batch.close()
    beam = counts[0] - 9  # the beam model's forms: 1 (fused) or 2 (two-pass)
    assert beam in (1, 2) and counts == [counts[0]] * len(counts), counts


def toy_model(states):
    import torch

    return torch.exp(-(states[:, 2] * states[:, 2] + states[:, 3] * states[:, 3]) / 10.0)


def lo_factors(states, det, pos, cat):
    lmap = lo.LandmarkMap([(*p, c) for p, c in zip(pos.tolist(), cat.tolist())])
    dets = [(*p, c) for p, c in zip(det[0].tolist(), det[1].tolist())]
    return np.array([lo.landmark_weight(s, dets, lmap, *SIGMA) for s in states.tolist()])


def test_factors_match_the_oracle(bb):
    """A member's weights after a normalising step are its propagated states' oracle likelihoods, normalised, to 1e-11."""
    rng = np.random.default_rng(23)
    pos, cat = random_map(rng, 500, 3)
    params = [bb.AmclParams(update_min_d=0.0, update_min_a=0.0, resample_interval=1000, min_particles=3000, max_particles=3000, seed=4)]
    f = Fleet(bb, params, [("landmark", bb.LandmarkMap(pos, cat))], [0])
    det = random_detections(rng, 40, 3)
    got, _ = f.step(0, [det])
    assert got[0].updated == 1 and got[0].resampled == 0
    states, w = f.batch.particles(0)
    want = lo_factors(states, det, pos, cat)
    np.testing.assert_allclose(w, want / want.sum(), rtol=1e-11, atol=0.0)


def test_map_moves_and_state_blobs(bb):
    """update_map from a grid map to a landmark map and back mid-trajectory, and a landmark member exported from a
    standalone filter into the batch and back: every step continues byte-identically."""
    sc = lfm_scene(bb)
    rng = np.random.default_rng(29)
    pos, cat = random_map(rng, 60, 4)
    lmap, grid = bb.LandmarkMap(pos, cat), bb.OccupancyGrid(sc.cells, sc.resolution)
    params = [bb.AmclParams(update_min_d=0.0, update_min_a=0.0, min_particles=800, max_particles=800, seed=7 + m, record_ancestors=True)
              for m in range(2)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION)] * 2, params)
    g = batch.add_likelihood_field_map(bb.LikelihoodFieldModelParam(), grid)
    lid = batch.add_landmark_map(model_param(bb, "landmark"), lmap)
    twins = [bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), p) for p in params]
    for m in range(2):
        batch.update_map(m, g)
        twins[m].update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(), grid)
        batch.initialize(m, sc.initial_mean, sc.initial_cov)
        twins[m].initialize(sc.initial_mean, sc.initial_cov)
    on_landmarks = [False, False]
    for t in range(1, 6):
        if t == 2 or t == 4:  # member 0 moves between the maps
            on_landmarks[0] = not on_landmarks[0]
            batch.update_map(0, lid if on_landmarks[0] else g)
            if on_landmarks[0]:
                twins[0].update_map(bb.SENSOR_LANDMARK, model_param(bb, "landmark"), lmap)
            else:
                twins[0].update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(), grid)
        x, y, th = sc.poses[t]
        poses = np.stack([[math.cos(th), math.sin(th), x, y]] * 2)
        dets = [random_detections(rng, 5, 4) for _ in range(2)]
        meas = [bb.Detections(*dets[m]) if on_landmarks[m] else sc.scans[t] for m in range(2)]
        got = batch.update_measurements(poses, meas)
        for m in range(2):
            exp = twins[m].update_landmarks(poses[m], *dets[m]) if on_landmarks[m] else twins[m].update(poses[m], sc.scans[t])
            assert_twin(batch, m, twins[m], got[m], exp, (t, m))

    # a standalone landmark filter joins the batch, steps there, and leaves again
    solo = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), params[1])
    solo.update_map(bb.SENSOR_LANDMARK, model_param(bb, "landmark"), lmap)
    solo.initialize([0.0, 0.0, 0.0], np.diag([0.5, 0.5, 0.2]))
    twin = bb.Amcl.from_state(solo.export_state())
    twin.update_map(bb.SENSOR_LANDMARK, model_param(bb, "landmark"), lmap)
    slot = batch.import_member(solo.export_state(), lid)
    for t in range(3):
        det = random_detections(rng, 7, 4)
        pose = np.array([math.cos(0.2 * t), math.sin(0.2 * t), 0.3 * t, 0.0])
        poses = np.stack([pose] * len(batch))
        present = [m == slot for m in range(len(batch))]
        meas = [bb.Detections(*det) if m == slot else None for m in range(len(batch))]
        got = batch.update_measurements(poses, meas, present)
        assert_twin(batch, slot, twin, got[slot], twin.update_landmarks(pose, *det), t)
    back = bb.Amcl.from_state(batch.export_member(slot))
    back.update_map(bb.SENSOR_LANDMARK, model_param(bb, "landmark"), lmap)
    det = random_detections(rng, 7, 4)
    ra, rb = back.update_landmarks([1.0, 0.0, 1.5, 0.0], *det), twin.update_landmarks([1.0, 0.0, 1.5, 0.0], *det)
    assert result_bytes(ra) == result_bytes(rb) and back.particles()[0].tobytes() == twin.particles()[0].tobytes()


def test_members_join_and_leave_around_landmark_members(bb):
    rng = np.random.default_rng(31)
    pos, cat = random_map(rng, 80, 4)
    maps = [("landmark", bb.LandmarkMap(pos, cat)), ("bearing", bb.LandmarkMap(pos, cat))]
    params = fleet_params(bb, "systematic", (600, 900, 300))
    f = Fleet(bb, params, maps, [0, 1, 0])
    f.step(0, [random_detections(rng, 4, 4) for _ in range(3)])
    f.batch.remove_member(1)
    # a removed member's staged detections go with it: its successor must stage its own
    new = bb.AmclParams(update_min_d=0.05, update_min_a=0.05, min_particles=500, max_particles=500, seed=99, record_ancestors=True)
    slot = f.batch.add_member(bb.DifferentialDriveModelParam(*MOTION), new)
    assert slot == 1
    f.batch.update_map(1, 0)
    f.batch.initialize(1, [0.0, 0.0, 0.0], np.diag([0.3, 0.3, 0.1]))
    twin = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), new)
    twin.update_map(bb.SENSOR_LANDMARK, model_param(bb, "landmark"), bb.LandmarkMap(pos, cat))
    twin.initialize([0.0, 0.0, 0.0], np.diag([0.3, 0.3, 0.1]))
    f.twins[1] = twin
    for t in range(1, 4):
        f.step(t, [random_detections(rng, 5, 4) for _ in range(3)])


def test_refusals_leave_every_member_unchanged(bb):
    from beluga_b200 import BelugaB200Error, _capi
    import ctypes as C

    sc = lfm_scene(bb)
    rng = np.random.default_rng(37)
    pos, cat = random_map(rng, 30, 3)
    lmap, grid = bb.LandmarkMap(pos, cat), bb.OccupancyGrid(sc.cells, sc.resolution)
    params = [bb.AmclParams(update_min_d=0.0, update_min_a=0.0, min_particles=200, max_particles=200, seed=m) for m in range(3)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION)] * 3, params)
    lid = batch.add_landmark_map(model_param(bb, "landmark"), lmap)
    g = batch.add_likelihood_field_map(bb.LikelihoodFieldModelParam(), grid)
    for m, i in enumerate((lid, lid, g)):
        batch.update_map(m, i)
        batch.initialize(m, [0.0, 0.0, 0.0], np.diag([0.3, 0.3, 0.1]))
    blobs = batch.export_members()
    lib, h = batch._lib, batch._h
    poses = np.stack([[1.0, 0.0, 0.2, 0.0]] * 3)
    det = random_detections(rng, 3, 3)

    def refused(call, status):
        with pytest.raises(BelugaB200Error) as e:
            call()
        assert e.value.status == status
        assert batch.export_members() == blobs

    # member 1 never had detections staged
    refused(lambda: lib_update(batch, poses, [_capi.MEASUREMENT_LANDMARKS] * 2 + [_capi.MEASUREMENT_POINTS]), STATE)
    batch.update_measurements(poses, [bb.Detections(*det), bb.Detections(*det), sc.scans[1]], present=[0, 0, 1])  # no staging: absent
    blobs = batch.export_members()
    refused(lambda: batch.update_measurements(poses, [bb.Detections(*det), sc.scans[1], sc.scans[1]]), STATE)  # points on a landmark map
    refused(lambda: batch.update_measurements(poses, [bb.Detections(*det)] * 3), STATE)  # detections on a grid map
    refused(lambda: batch.update_clustered(poses, [bb.Detections(*det)] * 3), STATE)
    refused(lambda: batch.update_weighted(poses, [bb.Detections(*det), None, bb.Detections(*det)], lambda *a: None), STATE)
    refused(lambda: batch.likelihood_field(lid), STATE)
    bear = np.array([[1.0, 0.0]])
    refused(lambda: batch.cast_rays([np.array([[1.0, 0.0, 0.0, 0.0]])] * 3, bear, 5.0, present=[1, 0, 0]), STATE)
    refused(lambda: batch.cast_rays([np.array([[1.0, 0.0, 0.0, 0.0]])] * 3, bear, 5.0, present=[0, 0, 1], map_ids=[-1, -1, lid]), STATE)
    # set_detections: null arrays with a count, too many, a vacant slot
    n = (C.c_uint64 * 3)(1, 0, 0)
    assert lib.bb200_amcl_batch_set_detections(h, None, n, None) == INVALID
    ptrs = (C.POINTER(_capi.Landmark) * 3)(None, None, None)
    assert lib.bb200_amcl_batch_set_detections(h, ptrs, n, None) == INVALID
    assert lib.bb200_amcl_batch_set_detections(h, ptrs, (C.c_uint64 * 3)(0, 0xFFFFFFFF, 0), None) == INVALID
    # parameter and map errors: the standalone filter's statuses and messages
    f = bb.Filter(capacity=16)
    bad = [(bb.LandmarkModelParam(0.0, 1.0, 0.1), None), (bb.LandmarkModelParam(1.0, 1.0, 1.5), None), (None, bb.BearingModelParam(-1.0)),
           (None, bb.BearingModelParam(1.0, np.diag([1.0, 1.0, -1.0, 0.0])[:3]))]
    for lp, bp in bad:
        with pytest.raises(BelugaB200Error) as want:
            f.set_landmark_map(lp, lmap) if lp is not None else f.set_bearing_map(bp, lmap)
        with pytest.raises(BelugaB200Error) as got:
            batch.add_landmark_map(lp, lmap) if lp is not None else batch.add_bearing_map(bp, lmap)
        assert (got.value.status, str(got.value)) == (want.value.status, str(want.value))
    assert batch.export_members() == blobs
    # with the refusals behind it, a step runs as on a fresh batch
    fresh = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION)] * 3, params)
    fid = fresh.add_landmark_map(model_param(bb, "landmark"), lmap)
    fg = fresh.add_likelihood_field_map(bb.LikelihoodFieldModelParam(), grid)
    for m, i in enumerate((fid, fid, fg)):
        fresh.update_map(m, i)
        fresh.initialize(m, [0.0, 0.0, 0.0], np.diag([0.3, 0.3, 0.1]))
    fresh.update_measurements(poses, [bb.Detections(*det), bb.Detections(*det), sc.scans[1]], present=[0, 0, 1])
    meas = [bb.Detections(*det), bb.Detections(*det), sc.scans[2]]
    ra, rb = batch.update_measurements(poses, meas), fresh.update_measurements(poses, meas)
    assert [result_bytes(r) for r in ra] == [result_bytes(r) for r in rb]


def lib_update(batch, poses, kinds):
    """bb200_amcl_batch_update_measurements with bare kinds (no staging through the Python wrapper)."""
    from beluga_b200 import _capi, _dptr

    k = len(kinds)
    pts = np.zeros((1, 2))
    table = (_capi.Measurement * k)(*[_capi.Measurement(kind=c, points_xy=_dptr(pts), n_points=1) for c in kinds])
    res = (_capi.UpdateResult * k)()
    batch._check(batch._lib.bb200_amcl_batch_update_measurements(batch._h, _dptr(np.ascontiguousarray(poses)), table, None, res))
