"""Landmark and bearing steps on a sharded filter without a GPU: the new entry points' declarations, exports and ctypes table,
their refusals of null handles and arguments, and a sharded filter that cannot be created without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NO_DEVICE = -1, -3
NEW = ["bb200_sharded_amcl_set_landmark_map", "bb200_sharded_amcl_set_bearing_map", "bb200_sharded_amcl_update_landmarks"]


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_symbols_declared_exported_and_wrapped(lib):
    from beluga_b200 import _capi

    with open(os.path.join(ROOT, "include", "beluga_b200.h")) as f:
        header = f.read()
    for decl in [r"int bb200_sharded_amcl_set_landmark_map\(bb200_sharded_amcl\* g, const bb200_landmark_param\* p, const bb200_landmark_map\* map\);",
                 r"int bb200_sharded_amcl_set_bearing_map\(bb200_sharded_amcl\* g, const bb200_bearing_param\* p, const bb200_landmark_map\* map\);",
                 r"int bb200_sharded_amcl_update_landmarks\(bb200_sharded_amcl\* g, const double control_pose\[4\], const bb200_landmark_detection\* detections, "
                 r"uint64_t n,\s+bb200_update_result\* out\);"]:
        assert re.search(decl, header), decl
    assert "#define BB200_ABI_VERSION 2" in header
    for name in NEW:
        assert name in _capi.SIGNATURES
        assert getattr(lib, name) is not None


def test_calls_without_a_filter_fail_cleanly(lib):
    from beluga_b200 import _capi

    pose = np.array([1.0, 0.0, 0.0, 0.0])
    pose_p = pose.ctypes.data_as(C.POINTER(C.c_double))
    res = _capi.UpdateResult()
    lp, bp = _capi.LandmarkParam(1.0, 1.0, 1e-4), _capi.BearingParam()
    det = (_capi.Landmark * 1)()
    lmap = _capi.LandmarkMap(det, 1, None, None)
    assert lib.bb200_sharded_amcl_set_landmark_map(None, C.byref(lp), C.byref(lmap)) == INVALID
    assert lib.bb200_sharded_amcl_set_bearing_map(None, C.byref(bp), C.byref(lmap)) == INVALID
    assert lib.bb200_sharded_amcl_update_landmarks(None, pose_p, det, 1, C.byref(res)) == INVALID
    # Every other argument is checked too, before the handle is read: any pointer stands in for a filter here.
    fake = C.c_void_p(C.addressof(res))
    assert lib.bb200_sharded_amcl_set_landmark_map(fake, None, C.byref(lmap)) == INVALID
    assert lib.bb200_sharded_amcl_set_landmark_map(fake, C.byref(lp), None) == INVALID
    assert lib.bb200_sharded_amcl_set_bearing_map(fake, None, C.byref(lmap)) == INVALID
    assert lib.bb200_sharded_amcl_set_bearing_map(fake, C.byref(bp), None) == INVALID
    assert lib.bb200_sharded_amcl_update_landmarks(fake, None, det, 1, C.byref(res)) == INVALID
    assert lib.bb200_sharded_amcl_update_landmarks(fake, pose_p, det, 1, None) == INVALID
    assert lib.bb200_sharded_amcl_update_landmarks(fake, pose_p, None, 3, C.byref(res)) == INVALID


def test_sharded_filter_needs_a_device(lib):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.ShardedAmcl(bb.DifferentialDriveModelParam(), bb.AmclParams(min_particles=16, max_particles=16), devices=[0, 0])
    assert e.value.status == NO_DEVICE
    assert callable(bb.ShardedAmcl.update_landmarks)
