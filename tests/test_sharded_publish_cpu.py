"""A sharded filter's node cycle without a GPU: the new entry points' declarations, exports and ctypes table, their refusals of
null handles and arguments, and a sharded filter that cannot be created without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NO_DEVICE = -1, -3
NEW = ["bb200_sharded_amcl_update_scan", "bb200_sharded_amcl_update_point_cloud", "bb200_sharded_amcl_particle_histogram",
       "bb200_sharded_amcl_sample_states", "bb200_sharded_amcl_cast_rays"]


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
    for decl in [r"int bb200_sharded_amcl_update_scan\(bb200_sharded_amcl\* g, const double control_pose\[4\], const bb200_laser_scan\* scan, "
                 r"bb200_update_result\* out\);",
                 r"int bb200_sharded_amcl_update_point_cloud\(bb200_sharded_amcl\* g, const double control_pose\[4\], const bb200_point_cloud\* cloud,"
                 r"\s+bb200_update_result\* out\);",
                 r"int bb200_sharded_amcl_particle_histogram\(bb200_sharded_amcl\* g, double linear_resolution, double angular_resolution, "
                 r"bb200_cluster_cell\* bins,\s+uint64_t capacity, uint64_t\* n_bins, double\* max_bin_weight\);",
                 r"int bb200_sharded_amcl_sample_states\(bb200_sharded_amcl\* g, uint64_t count, uint32_t step, double\* states_out\);",
                 r"int bb200_sharded_amcl_cast_rays\(bb200_sharded_amcl\* g, const double\* poses, uint64_t n_poses, const double\* bearings_cs, "
                 r"uint64_t n_bearings,\s+double max_range, double\* ranges\);"]:
        assert re.search(decl, header), decl
    assert "#define BB200_ABI_VERSION 2" in header
    for name in NEW:
        assert name in _capi.SIGNATURES
        assert getattr(lib, name) is not None


def test_calls_without_a_filter_fail_cleanly(lib):
    from beluga_b200 import _capi

    d = C.POINTER(C.c_double)
    one = np.zeros(4)
    pose = one.ctypes.data_as(d)
    res = _capi.UpdateResult()
    scan = _capi.LaserScan()
    cloud = _capi.PointCloud()
    assert lib.bb200_sharded_amcl_update_scan(None, pose, C.byref(scan), C.byref(res)) == INVALID
    assert lib.bb200_sharded_amcl_update_point_cloud(None, pose, C.byref(cloud), C.byref(res)) == INVALID
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert lib.bb200_sharded_amcl_particle_histogram(None, 0.1, 0.1, None, 0, C.byref(n), C.byref(top)) == INVALID
    assert lib.bb200_sharded_amcl_sample_states(None, 1, 0, pose) == INVALID
    assert lib.bb200_sharded_amcl_cast_rays(None, pose, 1, pose, 1, 1.0, pose) == INVALID


def test_sharded_filter_needs_a_device(lib):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.ShardedAmcl(bb.DifferentialDriveModelParam(), bb.AmclParams(min_particles=16, max_particles=16), devices=[0, 0])
    assert e.value.status == NO_DEVICE
    for name in ("update_scan", "update_point_cloud", "particle_histogram", "sample_states", "cast_rays"):
        assert callable(getattr(bb.ShardedAmcl, name))
