"""Ray casts without a GPU: the new entry points' declarations, exports and ctypes table, their refusals of null handles, and
bb200_scan_bearings, which must give exactly the beam directions bb200_scan_to_points uses."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NO_DEVICE, CAPACITY = -1, -3, -5
NEW = ["bb200_filter_cast_rays", "bb200_amcl_batch_cast_rays", "bb200_scan_bearings"]


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
    for decl in [r"int bb200_filter_cast_rays\(bb200_filter\* f, const double\* poses, uint64_t n_poses, const double\* bearings_cs, "
                 r"uint64_t n_bearings, double max_range,\s+double\* ranges\);",
                 r"int bb200_amcl_batch_cast_rays\(bb200_amcl_batch\* b, const uint8_t\* present, const int\* map_ids, const double\* const\* poses, "
                 r"const uint64_t\* n_poses,\s+const double\* const\* bearings_cs, const uint64_t\* n_bearings, const double\* max_range, "
                 r"double\* const\* ranges\);",
                 r"int bb200_scan_bearings\(float angle_min, float angle_increment, uint64_t n_ranges, uint64_t max_beams, double\* bearings_cs, "
                 r"uint64_t capacity,\s+uint64_t\* n\);"]:
        assert re.search(decl, header), decl
    for name in NEW:
        assert name in _capi.SIGNATURES
        assert getattr(lib, name) is not None


def test_calls_without_a_device_fail_cleanly(lib):
    import beluga_b200 as bb

    d = C.POINTER(C.c_double)
    one = np.zeros(4)
    assert lib.bb200_filter_cast_rays(None, one.ctypes.data_as(d), 1, one.ctypes.data_as(d), 1, 1.0, one.ctypes.data_as(d)) == INVALID
    k = 1
    ptrs = (d * k)(one.ctypes.data_as(d))
    counts = (C.c_uint64 * k)(1)
    assert lib.bb200_amcl_batch_cast_rays(None, None, None, ptrs, counts, ptrs, counts, (C.c_double * k)(1.0), ptrs) == INVALID
    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.Filter(capacity=16)
    assert e.value.status == NO_DEVICE
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch([bb.DifferentialDriveModelParam()], [bb.AmclParams(min_particles=16, max_particles=16)])
    assert e.value.status == NO_DEVICE


@pytest.mark.parametrize("max_beams", [0, 1, 2, 7, 60, 359, 360, 361, 1000])
@pytest.mark.parametrize("n_ranges", [0, 1, 360])
def test_scan_bearings_equal_scan_to_points_directions(lib, n_ranges, max_beams):
    import beluga_b200 as bb

    angle_min, angle_increment = np.float32(-math.pi), np.float32(2 * math.pi / 360)
    # unit ranges, all valid, identity origin: each point is exactly the beam's (cos, sin)
    points = bb.scan_to_points(np.ones(n_ranges, np.float32), float(angle_min), float(angle_increment), max_beams=max_beams)
    bearings = bb.scan_bearings(float(angle_min), float(angle_increment), n_ranges, max_beams)
    assert bearings.shape == points.shape
    assert bearings.tobytes() == points.tobytes()


def test_scan_bearings_size_query_and_capacity(lib):
    n = C.c_uint64(0)
    assert lib.bb200_scan_bearings(0.0, 0.01, 100, 30, None, 0, C.byref(n)) == CAPACITY and n.value == 30
    out = np.full((29, 2), 7.0)
    assert lib.bb200_scan_bearings(0.0, 0.01, 100, 30, out.ctypes.data_as(C.POINTER(C.c_double)), 29, C.byref(n)) == CAPACITY
    assert (out == 7.0).all()  # nothing written
    assert lib.bb200_scan_bearings(0.0, 0.01, 100, 30, None, 5, C.byref(n)) == INVALID
    assert lib.bb200_scan_bearings(0.0, 0.01, 100, 30, None, 0, None) == INVALID
    assert lib.bb200_scan_bearings(0.0, 0.01, 0, 30, None, 0, C.byref(n)) == 0 and n.value == 0
