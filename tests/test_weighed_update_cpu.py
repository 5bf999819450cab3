"""The weighed step's surface without a device: bb200_amcl_update_begin / _end are declared and exported with their
view struct, refuse null handles and arguments, and the Python entry point refuses to run without a GPU."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import build as bb_build
    from beluga_b200 import _capi

    bb_build.build()
    return _capi.load()


def test_header_declares_the_view_and_both_halves():
    text = open(os.path.join(ROOT, "include", "beluga_b200.h")).read()
    assert re.search(r"typedef struct bb200_weigh_view \{.*?\} bb200_weigh_view;", text, flags=re.S)
    assert "int bb200_amcl_update_begin(bb200_amcl* a, const double control_pose[4], bb200_weigh_view* view);" in text
    assert "int bb200_amcl_update_end(bb200_amcl* a, bb200_update_result* out);" in text


def test_view_layout_matches_the_header(lib):
    from beluga_b200 import _capi

    v = _capi.WeighView
    assert [f for f, _ in v._fields_] == ["updated", "n", "states", "factors", "stream"]
    assert C.sizeof(v) == 40 and v.n.offset == 8 and v.stream.offset == 32


def test_null_arguments_are_refused(lib):
    from beluga_b200 import _capi

    view, res = _capi.WeighView(), _capi.UpdateResult()
    pose = (C.c_double * 4)(1.0, 0.0, 0.0, 0.0)
    assert lib.bb200_amcl_update_begin(None, pose, C.byref(view)) == -1
    assert lib.bb200_amcl_update_end(None, C.byref(res)) == -1


def test_no_cpu_fallback(lib):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    assert hasattr(bb.Amcl, "update_weighted")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.Amcl(bb.DifferentialDriveModelParam(), bb.AmclParams())
    assert e.value.status == -3  # BB200_ERR_NO_DEVICE
