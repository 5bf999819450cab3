"""Several maps in one batch without a GPU: every new entry point (add_*_map, update_map, member_map, remove_map,
get_likelihood_field) refuses a null handle with BB200_ERR_INVALID_ARGUMENT, whatever the other arguments are, and writes
nothing; the ctypes table and AmclBatch carry the entry points, and the ABI version stays 2.  The null arguments with a
real handle need a batch, hence a device: tests/test_gpu_batch_maps.py checks them."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_null_handle(lib):
    import beluga_b200 as bb

    lfm = bb.LikelihoodFieldModelParam().c()
    beam = bb.BeamModelParam().c()
    g = bb.OccupancyGrid(np.zeros((4, 4), dtype=np.int8), 0.05).c()
    i = C.c_int(-7)
    out = np.zeros(16, dtype=np.float32)
    fp = out.ctypes.data_as(C.POINTER(C.c_float))
    for prob in (0, 1):
        assert lib.bb200_amcl_batch_add_likelihood_field_map(None, C.byref(lfm), C.byref(g), prob, C.byref(i)) == -1
        assert lib.bb200_amcl_batch_add_likelihood_field_map(None, None, C.byref(g), prob, C.byref(i)) == -1
        assert lib.bb200_amcl_batch_add_likelihood_field_map(None, C.byref(lfm), None, prob, C.byref(i)) == -1
        assert lib.bb200_amcl_batch_add_likelihood_field_map(None, C.byref(lfm), C.byref(g), prob, None) == -1
    assert lib.bb200_amcl_batch_add_beam_map(None, C.byref(beam), C.byref(g), C.byref(i)) == -1
    assert lib.bb200_amcl_batch_add_beam_map(None, None, C.byref(g), C.byref(i)) == -1
    assert lib.bb200_amcl_batch_add_beam_map(None, C.byref(beam), None, C.byref(i)) == -1
    assert lib.bb200_amcl_batch_add_beam_map(None, C.byref(beam), C.byref(g), None) == -1
    assert lib.bb200_amcl_batch_update_map(None, 0, 0) == -1
    assert lib.bb200_amcl_batch_member_map(None, 0, C.byref(i)) == -1
    assert lib.bb200_amcl_batch_member_map(None, 0, None) == -1
    assert lib.bb200_amcl_batch_remove_map(None, 0) == -1
    assert lib.bb200_amcl_batch_get_likelihood_field(None, 0, fp, out.size) == -1
    assert lib.bb200_amcl_batch_get_likelihood_field(None, 0, None, 0) == -1
    assert i.value == -7  # nothing written


def test_python_exposes_the_entry_points(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    vp, grid, ip = C.c_void_p, C.POINTER(_capi.OccupancyGrid), C.POINTER(C.c_int)
    assert _capi.SIGNATURES["bb200_amcl_batch_add_likelihood_field_map"] == (
        C.c_int, [vp, C.POINTER(_capi.LikelihoodFieldParam), grid, C.c_int, ip])
    assert _capi.SIGNATURES["bb200_amcl_batch_add_beam_map"] == (C.c_int, [vp, C.POINTER(_capi.BeamParam), grid, ip])
    assert _capi.SIGNATURES["bb200_amcl_batch_update_map"] == (C.c_int, [vp, C.c_int, C.c_int])
    assert _capi.SIGNATURES["bb200_amcl_batch_member_map"] == (C.c_int, [vp, C.c_int, ip])
    assert _capi.SIGNATURES["bb200_amcl_batch_remove_map"] == (C.c_int, [vp, C.c_int])
    assert _capi.SIGNATURES["bb200_amcl_batch_get_likelihood_field"] == (C.c_int, [vp, C.c_int, C.POINTER(C.c_float), C.c_uint64])
    for name in ("add_likelihood_field_map", "add_beam_map", "update_map", "member_map", "remove_map", "likelihood_field"):
        assert callable(getattr(bb.AmclBatch, name)), name
    assert lib.bb200_abi_version() == 2
