"""The landmark and bearing models without a GPU: the oracle of tests/_landmark_oracle.py on the reference's own gtest
cases, the kernel's per-particle body (csrc/reweight_landmark.cuh, through tests/cpp/landmark_probe.cpp) against the
oracle bit for bit, and the C ABI's refusals before any device call."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _landmark_oracle as lo  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "beluga_b200", "csrc")

# test/beluga/sensor/test_landmark_sensor_model.cpp: sigma_range 1, sigma_bearing pi/2, random_prob 1e-4, the robot at
# SE2d{SO2d{-pi/2}, {1, -1}}, map bounds [-10, 10]^2 x {0}.
SIG = (1.0, math.pi / 2.0, 1e-4)
POSE = (math.cos(-math.pi / 2.0), math.sin(-math.pi / 2.0), 1.0, -1.0)
BOUNDS = ((-10.0, -10.0, 0.0), (10.0, 10.0, 0.0))


def lw(landmarks, detections):
    return lo.landmark_weight(POSE, detections, lo.LandmarkMap(landmarks, BOUNDS), *SIG)


def test_gtest_bulls_eye_detection():  # BullsEyeDetection
    assert lw([(3.0, -2.0, 0.0, 0)], [(1.0, 2.0, 0.0, 0)]) == pytest.approx(1.0, abs=1e-2)


def test_gtest_map_update():  # MapUpdate: an empty map, then the landmark
    assert lw([], [(1.0, 2.0, 0.0, 0)]) == pytest.approx(0.0, abs=1e-2)
    assert lw([(3.0, -2.0, 0.0, 0)], [(1.0, 2.0, 0.0, 0)]) == pytest.approx(1.0, abs=1e-2)


def test_gtest_multiple_bulls_eye_detections():  # MultipleBullsEyeDetections
    lms = [(1.0, -2.0, 0.0, 0), (1.0, -0.0, 0.0, 1), (2.0, -1.0, 0.0, 2), (0.0, -1.0, 0.0, 3)]
    dets = [(1.0, 0.0, 0.0, 0), (-1.0, 0.0, 0.0, 1), (0.0, 1.0, 0.0, 2), (0.0, -1.0, 0.0, 3)]
    assert lw(lms, dets) == pytest.approx(1.0, abs=1e-2)


@pytest.mark.parametrize("det,want", [((10.0, 0.0, 0.0), 1.0), ((9.0, 0.0, 0.0), 0.6), ((11.0, 0.0, 0.0), 0.6)])
def test_gtest_one_std_in_range(det, want):  # OneStdInRange
    assert lw([(1.0, -11.0, 0.0, 0)], [(*det, 0)]) == pytest.approx(want, abs=1e-2)


@pytest.mark.parametrize("det,want", [((10.0, 0.0, 0.0), 1.0), ((0.0, 10.0, 0.0), 0.6), ((0.0, -10.0, 0.0), 0.6)])
def test_gtest_one_std_in_bearing(det, want):  # OneStdInBearing
    assert lw([(1.0, -11.0, 0.0, 0)], [(*det, 0)]) == pytest.approx(want, abs=1e-2)


def test_gtest_no_such_landmark():  # NoSuchLandmark
    assert lw([(0.0, 1.0, 0.0, 99)], [(0.0, 2.0, 0.0, 88)]) == pytest.approx(1e-4, abs=1e-6)


def test_bearing_bulls_eye_and_missing_category():
    # test_bearing_sensor_model.cpp's setting in spirit: a camera at the robot looking along x sees a landmark dead ahead
    m = lo.LandmarkMap([(3.0, 0.0, 0.0, 0)])
    assert lo.bearing_weight((1.0, 0.0, 0.0, 0.0), [(1.0, 0.0, 0.0, 0)], m, 1.0, lo.IDENTITY_POSE) == 1.0
    assert lo.bearing_weight((1.0, 0.0, 0.0, 0.0), [(1.0, 0.0, 0.0, 1)], m, 1.0, lo.IDENTITY_POSE) == 0.0
    # a right angle off the landmark: exp(-(pi/2)^2 / 2)
    got = lo.bearing_weight((1.0, 0.0, 0.0, 0.0), [(0.0, 1.0, 0.0, 0)], m, 1.0, lo.IDENTITY_POSE)
    assert got == pytest.approx(math.exp(-(math.pi / 2) ** 2 / 2), rel=1e-15)


BEARING_MAP = [(9.0, 0.0, 1.0, 0), (0.0, 9.0, 1.0, 0), (0.0, 0.0, 9.0, 0), (-9.0, 0.0, 1.0, 1), (0.0, -9.0, 1.0, 1), (0.0, 0.0, -9.0, 1),
               (0.0, 0.0, -9.0, 2)]  # test_landmark_map.cpp LandmarkMapBearingTest, sensor at (0, 0, 1)
SENSOR_AT_1 = ((1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 1.0))


def test_gtest_bearing_map_limits():  # LandmarkMapBearingTest.MapLimits
    m = lo.LandmarkMap(BEARING_MAP, ((0.0, 1.0, 2.0), (10.0, 11.0, 12.0)))
    assert m.map_limits() == ((0.0, 1.0, 2.0), (10.0, 11.0, 12.0))


@pytest.mark.parametrize("detection,category,want", [
    ((1.0, 0.0, 0.0), 0, (1.0, 0.0, 0.0)),     # TrivialQuery1
    ((-1.0, 0.0, 0.0), 1, (-1.0, 0.0, 0.0)),   # TrivialQuery2
    ((1.0, 0.0, 0.0), 2, (0.0, 0.0, -1.0)),    # FeatureInTotallyDifferentDirection
])
def test_gtest_bearing_queries(detection, category, want):
    got = lo.LandmarkMap(BEARING_MAP).find_closest_bearing_landmark(detection, category, SENSOR_AT_1)
    assert math.dist(got, want) < 1e-6


def test_gtest_bearing_no_such_feature():  # LandmarkMapBearingTest.NoSuchFeature
    assert lo.LandmarkMap(BEARING_MAP).find_closest_bearing_landmark((1.0, 0.0, 0.0), 99, SENSOR_AT_1) is None


def test_gtest_bounding_region_2d():  # test_multivariate_uniform_distribution.cpp BoundingRegion2d
    from oracle import pyoracle

    pyoracle.build()
    box = (3.0, 3.0 + 0.01, -2.0, -2.0 + 0.01)
    for index in range(200):
        _, x, y = lo.box_state(1234, index, 0, box, pyoracle.philox4x32_10)
        assert abs(x - 3.0) <= 0.01 and abs(y + 2.0) <= 0.01


def test_map_limits():  # test_landmark_map.cpp: explicit, implicit and empty limits
    lms = [(1.0, -2.0, 3.0, 0), (-4.0, 5.0, -6.0, 1), (7.0, 0.0, 0.5, 0)]
    assert lo.LandmarkMap(lms, BOUNDS).map_limits() == BOUNDS
    assert lo.LandmarkMap(lms).map_limits() == ((-4.0, -2.0, -6.0), (7.0, 5.0, 3.0))
    lo_, hi = lo.LandmarkMap([]).map_limits()
    assert all(a > b for a, b in zip(lo_, hi))  # an empty box


def test_first_minimum_wins():
    m = lo.LandmarkMap([(1.0, 0.0, 0.0, 0), (-1.0, 0.0, 0.0, 0), (0.0, 1.0, 0.0, 0)])
    assert m.find_nearest_landmark((0.0, 0.0, 0.0), 0) == (1.0, 0.0, 0.0)
    assert m.find_nearest_landmark((0.0, 0.0, 0.0), 1) is None
    m = lo.LandmarkMap([(2.0, 0.0, 0.0, 0), (1.0, 0.0, 0.0, 0), (float("nan"), 0.0, 0.0, 0)])
    frame = lo.robot_frame((1.0, 0.0, 0.0, 0.0))
    assert m.find_closest_bearing_landmark((1.0, 0.0, 0.0), 0, frame) == (1.0, 0.0, 0.0)


def test_product_grouping():
    v = [0.1 * k + 0.3 for k in range(11)]
    want = 1.0 * ((v[0] * v[1]) * (v[2] * v[3]))
    want = want * ((v[4] * v[5]) * (v[6] * v[7]))
    want = ((want * v[8]) * v[9]) * v[10]
    assert lo.product_by_fours(v) == want


# ---- the kernel's per-particle body against the oracle, bit for bit ---------------------------------------------------


def make_case(rng, model, kind):
    n_cat = int(rng.choice([1, 3, 64]))
    n_lm = int(rng.integers(0, 40))
    grid = kind == "ties"
    if grid:  # integer coordinates: exact distance ties, duplicates, landmarks on rays from the sensor
        lms = rng.integers(-3, 4, (n_lm, 3)).astype(float)
        lms[:, 2] = rng.integers(0, 2, n_lm)
    else:
        lms = rng.uniform(-20, 20, (n_lm, 3))
    cats = rng.integers(0, n_cat, n_lm).astype(float)
    n_det = int(rng.integers(0, 10))
    dets = rng.integers(-3, 4, (n_det, 3)).astype(float) if grid else rng.uniform(-5, 5, (n_det, 3))
    if n_det:
        dets[rng.random(n_det) < 0.15] = 0.0  # zero-length detections
    dcat = rng.integers(0, n_cat + 1, n_det).astype(float)  # category n_cat: none in the map
    n = 8
    th = rng.uniform(-np.pi, np.pi, n)
    st = np.stack([np.cos(th), np.sin(th), rng.uniform(-20, 20, n), rng.uniform(-20, 20, n)], axis=1)
    if grid:
        st[:, :2] = [[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]][rng.integers(0, 4)]
        st[:, 2:] = rng.integers(-3, 4, (n, 2))
    if kind == "edge":
        st[0] = [np.nan, 0.0, 0.0, 0.0]
        st[1] = [1.0, 0.0, 1e300, -1e300]
        st[2] = [0.6, 0.8, np.nan, 1.0]
        st[3] = [1.0, 0.0, 5e15, 5e15]
        if n_lm:
            st[4, 2:] = lms[0, :2]  # a landmark at the particle
    sigma = (float(rng.uniform(0.1, 2.0)), float(rng.uniform(0.1, 2.0)), float(rng.uniform(0.0, 0.1)))
    if model == lo_bearing:
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        q = q * np.sign(np.linalg.det(q))
        pose = np.concatenate([q, rng.uniform(-1, 1, (3, 1))], axis=1).reshape(12)
        if grid:
            pose = np.array(lo.IDENTITY_POSE)
    else:
        pose = np.array(lo.IDENTITY_POSE)
    return st, np.concatenate([dets, dcat[:, None]], axis=1), np.concatenate([lms, cats[:, None]], axis=1), sigma, pose


lo_landmark, lo_bearing = 3, 4


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("landmark_probe") / "probe")  # the checkout may be read-only
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror", "-Wno-unknown-pragmas", "-I", CSRC,
           os.path.join(ROOT, "tests", "cpp", "landmark_probe.cpp"), "-o", exe]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-4000:]
    return exe


@pytest.mark.parametrize("model", [lo_landmark, lo_bearing])
@pytest.mark.parametrize("kind", ["random", "ties", "edge"])
def test_kernel_body_matches_oracle_bit_for_bit(probe, tmp_path, model, kind):
    rng = np.random.default_rng(model * 10 + len(kind))
    cases = [make_case(rng, model, kind) for _ in range(700)]
    blob = []
    for st, det, lms, sigma, pose in cases:
        head = [model, len(st), len(det), len(lms), *sigma, *pose]
        blob.append(np.concatenate([np.array(head, dtype=float), st.reshape(-1), det.reshape(-1), lms.reshape(-1)]))
    (tmp_path / "in.bin").write_bytes(np.concatenate(blob).tobytes())
    run = subprocess.run([probe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr
    got = np.frombuffer((tmp_path / "out.bin").read_bytes(), dtype=np.float64)
    want = []
    for st, det, lms, sigma, pose in cases:
        m = lo.LandmarkMap([tuple(r[:3]) + (int(r[3]),) for r in lms.tolist()])
        d = [tuple(r[:3]) + (int(r[3]),) for r in det.tolist()]
        for s in st.tolist():
            if model == lo_landmark:
                want.append(lo.landmark_weight(s, d, m, *sigma))
            else:
                want.append(lo.bearing_weight(s, d, m, sigma[1], tuple(pose.tolist())))
    want = np.array(want)
    assert len(got) == len(want) == 700 * 8
    same = (got.view(np.uint64) == want.view(np.uint64)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), (np.flatnonzero(~same)[:5], got[~same][:5], want[~same][:5])
    assert np.isfinite(want).sum() > len(want) // 2  # the cases weigh, not just fail


# ---- C ABI without a device ---------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_capi_refuses_without_a_device_or_with_null_arguments(lib):
    from beluga_b200 import _capi

    if lib.bb200_device_count() == 0:
        cfg = _capi.FilterConfig(0, 16, 0, 0, 0, 0)
        h = C.c_void_p()
        assert lib.bb200_filter_create(C.byref(cfg), C.byref(h)) == _capi.ERR_NO_DEVICE
    p = _capi.LandmarkParam(1.0, 1.0, 0.1)
    bp = _capi.BearingParam(1.0, (C.c_double * 12)(1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0))
    m = _capi.LandmarkMap(None, 0, None, None)
    r = _capi.UpdateResult()
    pose = (C.c_double * 4)(1, 0, 0, 0)
    inv = _capi.ERR_INVALID_ARGUMENT
    assert lib.bb200_filter_set_landmark_map(None, C.byref(p), C.byref(m)) == inv
    assert lib.bb200_filter_set_bearing_map(None, C.byref(bp), C.byref(m)) == inv
    assert lib.bb200_filter_reweight_landmarks(None, None, 0) == inv
    assert lib.bb200_amcl_update_landmarks(None, pose, None, 0, C.byref(r)) == inv


def test_python_surface(lib):
    import beluga_b200 as bb

    m = bb.LandmarkMap(np.zeros((2, 3)), [0, 1])
    assert m.c().n == 2 and not m.c().bounds_min3
    p = bb.BearingModelParam(0.5).c()
    assert list(p.sensor_pose_in_robot) == list(np.eye(3, 4).reshape(12))
    with pytest.raises(ValueError):
        bb.LandmarkMap(np.zeros((2, 3)), [0])


def test_map_argument_validation_on_the_host(lib, tmp_path):
    """prepare_landmark_map, the checks behind bb200_filter_set_landmark_map / _set_bearing_map, without a device:
    non-positive or non-finite sigmas, random_prob outside [0, 1], a sensor rotation that is not one within 1e-9, null
    landmarks with a count and half-given bounds are BB200_ERR_INVALID_ARGUMENT; the box is the bounds' or the landmarks'."""
    import shutil

    from beluga_b200 import build as bb_build

    cuda = os.path.dirname(os.path.dirname(os.path.realpath(shutil.which(bb_build.nvcc()))))
    lib_dir = os.path.join(ROOT, "beluga_b200")
    exe = str(tmp_path / "map_probe")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unknown-pragmas", "-I", CSRC, "-I", os.path.join(cuda, "include"),
           os.path.join(ROOT, "tests", "cpp", "landmark_map_probe.cpp"), "-o", exe, "-L", lib_dir, "-lbeluga_b200", f"-Wl,-rpath,{lib_dir}"]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-4000:]
    run = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert run.returncode == 0, run.stderr
    lines = run.stdout.split("\n")
    assert lines[:8] == ["landmark 0"] + ["landmark -1"] * 7
    assert lines[8:12] == ["bearing 0", "bearing -1", "bearing -1", "bearing -1"]
    assert lines[12:15] == ["map -1", "map -1", "map 0"]
    assert lines[15:18] == ["box -1 1 -1 1 1", "box -3 1 -2 4 1", "box - - - - 0"]
