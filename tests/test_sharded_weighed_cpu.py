"""The sharded weighed step's surface without a device: bb200_sharded_amcl_update_begin / _end are declared and exported,
refuse null handles and arguments, and ShardedAmcl.update_weighted exists with no CPU fallback."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import build as bb_build
    from beluga_b200 import _capi

    bb_build.build()
    return _capi.load()


def test_header_declares_both_halves():
    text = open(os.path.join(ROOT, "include", "beluga_b200.h")).read()
    assert "int bb200_sharded_amcl_update_begin(bb200_sharded_amcl* g, const double control_pose[4], bb200_weigh_view* views);" in text
    assert "int bb200_sharded_amcl_update_end(bb200_sharded_amcl* g, bb200_update_result* out);" in text


def test_both_halves_are_exported(lib):
    assert hasattr(lib, "bb200_sharded_amcl_update_begin") and hasattr(lib, "bb200_sharded_amcl_update_end")


def test_null_arguments_are_refused(lib):
    from beluga_b200 import _capi

    views, res = (_capi.WeighView * 2)(), _capi.UpdateResult()
    pose = (C.c_double * 4)(1.0, 0.0, 0.0, 0.0)
    assert lib.bb200_sharded_amcl_update_begin(None, pose, views) == -1
    assert lib.bb200_sharded_amcl_update_end(None, C.byref(res)) == -1


def test_no_cpu_fallback(lib):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    assert hasattr(bb.ShardedAmcl, "update_weighted")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.ShardedAmcl(bb.DifferentialDriveModelParam(), bb.AmclParams(min_particles=4000, max_particles=4000), devices=[0, 0])
    assert e.value.status == -3  # BB200_ERR_NO_DEVICE
