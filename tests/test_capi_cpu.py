"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports exactly the symbols that
include/beluga_b200.h declares, refuses to run without a GPU, and its host-only logic matches the oracle."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import build as bb_build
    from beluga_b200 import _capi

    bb_build.build()
    return _capi.load()


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "beluga_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bb200_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported(lib):
    from beluga_b200 import _capi

    out = subprocess.run(["nm", "-D", "--defined-only", _capi.LIB_PATH], check=True, capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (bb200_[a-z0-9_]+)", out))
    declared = declared_symbols()
    assert len(declared) >= 35
    missing = [s for s in declared if s not in exported]
    assert not missing, f"declared in include/beluga_b200.h but not exported: {missing}"
    undeclared = sorted(exported - set(declared))
    assert not undeclared, f"exported but not declared in include/beluga_b200.h: {undeclared}"
    assert set(_capi.SIGNATURES) == set(declared), "ctypes table and header disagree"
    assert lib.bb200_abi_version() == 2


def test_no_cpu_fallback(lib):
    """Without a CUDA device the product must fail loudly, never compute on the host."""
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.Filter(capacity=16)
    assert e.value.status == -3  # BB200_ERR_NO_DEVICE
    with pytest.raises(bb.BelugaB200Error):
        bb.Amcl(bb.DifferentialDriveModelParam(), bb.AmclParams())


def test_invalid_arguments_do_not_crash(lib):
    assert lib.bb200_filter_create(None, None) == -1
    assert lib.bb200_filter_size(None, None) == -1
    assert lib.bb200_last_error(None) == b"null filter"


@pytest.mark.parametrize(
    "pose,prev",
    [((1.0, 0.0, 0.0), (0.0, 0.0, 0.0)), ((0.0, 1.0, np.pi / 2), (0.0, 0.0, 0.0)), ((1.0, 2.0, -np.pi / 2), (0.0, 0.0, 0.0)),
     ((0.003, 0.002, 0.4), (0.0, 0.0, 0.1)), ((-1.0, -1.0, 0.0), (0.0, 0.0, 0.0)), ((5.3, -2.1, 2.9), (5.0, -2.0, -3.0))],
)
def test_diff_drive_sampling_matches_oracle(lib, orc, pose, prev):
    """Host part of DifferentialDriveModel::operator() (differential_drive_model.hpp:129-154)."""
    from beluga_b200 import _capi

    alphas = (0.1, 0.05, 0.1, 0.05)
    p = _capi.DiffDriveParam(*alphas, 0.01)
    a, b = orc.se2(*pose), orc.se2(*prev)
    out = _capi.DiffDriveSampling()
    assert lib.bb200_diff_drive_sampling_from_control(C.byref(p), a.ctypes.data_as(C.POINTER(C.c_double)),
                                                      b.ctypes.data_as(C.POINTER(C.c_double)), C.byref(out)) == 0
    got = np.array([out.rot1_mean, out.rot1_std, out.trans_mean, out.trans_std, out.rot2_mean, out.rot2_std])
    exp = orc.diff_drive_sampling(orc.MotionParam(*alphas), a, b)
    assert np.array_equal(got, exp)  # same libm, same operation order: bit-identical


@pytest.mark.parametrize("model", [0, 1, 2])
@pytest.mark.parametrize("pose,prev", [((1.0, 0.5, 0.3), (0.0, 0.0, 0.0)), ((0.001, 0.002, 1.4), (0.0, 0.0, 1.0)), ((-2.0, 3.0, -2.5), (-1.5, 2.0, 3.0))])
def test_motion_sampling_matches_oracle(lib, orc, model, pose, prev):
    """Host part of the three motion models (differential / omnidirectional / stationary)."""
    import beluga_b200 as bb

    alphas = (0.1, 0.05, 0.1, 0.05, 0.02)
    motion = [bb.DifferentialDriveModelParam(*alphas[:4]), bb.OmnidirectionalDriveModelParam(*alphas), bb.StationaryModelParam()][model]
    a, b = orc.se2(*pose), orc.se2(*prev)
    got = bb.motion_sampling(motion, a, b)
    exp = orc.motion_sampling(model, orc.OmniParam(*alphas), a, b)
    assert got.model == model
    assert np.array_equal(np.array(list(got.mean) + list(got.stddev) + list(got.first_rotation)), exp[:8])


@pytest.mark.parametrize(
    "size,count,expected",
    [(0, 0, []), (0, 1, []), (4, 0, []), (4, 1, [0]), (4, 10, [0, 1, 2, 3]), (4, 2, [0, 3]), (5, 3, [0, 2, 4]), (6, 3, [0, 3, 5]),
     (9, 3, [0, 4, 8]), (4, 3, [0, 2, 3]), (10, 6, [0, 2, 4, 6, 8, 9])],
)
def test_take_evenly_known_answers(lib, size, count, expected):
    """views/test_take_evenly.cpp:72-147 (inputs there are 1..size, so expected values are index + 1)."""
    import beluga_b200 as bb

    assert bb.take_evenly_indices(size, count).tolist() == expected


def test_scan_to_points(lib):
    """beluga_ros/test/test_laser_scan.cpp idea: range filter, NaN drop, beam subsampling, laser origin."""
    import beluga_b200 as bb

    ranges = np.array([0.05, 1.0, np.nan, 2.0, 50.0, 3.0, 4.0], dtype=np.float32)
    pts = bb.scan_to_points(ranges, angle_min=-0.5, angle_increment=0.25, min_range=0.1, max_range=10.0)
    keep = [1, 3, 5, 6]
    ang = (np.float32(-0.5) + np.arange(7, dtype=np.float32) * np.float32(0.25)).astype(np.float64)[keep]
    r = ranges[keep].astype(np.float64)
    assert np.array_equal(pts, np.stack([r * np.cos(ang), r * np.sin(ang)], axis=1))
    sub = bb.scan_to_points(ranges, -0.5, 0.25, 0.1, 10.0, max_beams=3)  # take_evenly(3) of 7 -> indices 0, 3, 6; index 0 is below min_range
    assert len(sub) == 2 and np.allclose(sub[0], [2.0 * np.cos(0.25), 2.0 * np.sin(0.25)])
    origin = np.array([[0.0, -1.0, 0.0, 0.3], [1.0, 0.0, 0.0, -0.2], [0.0, 0.0, 1.0, 0.5]])  # yaw 90 deg, offset
    moved = bb.scan_to_points(ranges, -0.5, 0.25, 0.1, 10.0, laser_origin=origin)
    assert np.allclose(moved, np.stack([-pts[:, 1] + 0.3, pts[:, 0] - 0.2], axis=1))


def test_scan_to_points_follows_the_reference_arithmetic():
    """bb200_scan_to_points against a numpy restatement of beluga_ros::LaserScan (beluga_ros/include/beluga_ros/laser_scan.hpp:69-80:
    take_evenly over ranges and angles, angle = float(angle_min + float(i) * angle_increment)), BaseLaserScan
    (beluga/sensor/data/laser_scan.hpp:64-91: drop NaN and out-of-range readings, x = r cos a, y = r sin a) and the laser origin
    transform of beluga_ros/src/amcl.cpp:57-62 -- bit for bit (the arithmetic is float32 angles widened to double)."""
    import beluga_b200 as bb

    rng = np.random.default_rng(6)
    n = 1081
    ranges = rng.uniform(0.05, 40.0, n).astype(np.float32)
    ranges[rng.integers(0, n, 40)] = np.nan
    ranges[rng.integers(0, n, 20)] = np.inf
    angle_min, angle_inc = np.float32(-2.35619449), np.float32(0.004363323)
    origin = np.array([[math.cos(0.3), -math.sin(0.3), 0.0, 0.25], [math.sin(0.3), math.cos(0.3), 0.0, -0.1], [0.0, 0.0, 1.0, 0.4]])
    for max_beams, use_origin in ((0, False), (60, False), (181, True), (5000, True)):
        got = bb.scan_to_points(ranges, float(angle_min), float(angle_inc), min_range=0.1, max_range=30.0, max_beams=max_beams,
                                laser_origin=origin if use_origin else None)
        count = n if max_beams == 0 else max_beams
        if count > n:
            idx = np.arange(n)
        else:  # take_evenly (views/take_evenly.hpp:118-145): first, last and evenly spaced in between, rounded up
            idx = np.array([0] + [-(-(p * (n - 1)) // (count - 1)) for p in range(1, count)], dtype=np.int64)
        exp = []
        for i in idx:
            r = float(ranges[i])
            theta = float(np.float32(angle_min + np.float32(np.float32(int(i)) * angle_inc)))
            if math.isnan(r) or not (r >= 0.1) or not (r <= 30.0):
                continue
            x, y = r * math.cos(theta), r * math.sin(theta)
            if use_origin:
                x, y = origin[0, 0] * x + origin[0, 1] * y + origin[0, 3], origin[1, 0] * x + origin[1, 1] * y + origin[1, 3]
            exp.append((x, y))
        assert np.array_equal(got, np.array(exp).reshape(-1, 2))
