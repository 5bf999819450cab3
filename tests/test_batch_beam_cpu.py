"""bb200_amcl_batch_set_beam_map without a GPU: a null handle or a null argument is refused with BB200_ERR_INVALID_ARGUMENT
before anything else is looked at; the ctypes table and AmclBatch carry the entry point."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_null_handle_and_null_arguments(lib):
    import beluga_b200 as bb

    p = bb.BeamModelParam().c()
    cells = np.zeros((4, 4), dtype=np.int8)
    g = bb.OccupancyGrid(cells, 0.05).c()
    assert lib.bb200_amcl_batch_set_beam_map(None, C.byref(p), C.byref(g)) == -1
    assert lib.bb200_amcl_batch_set_beam_map(None, None, None) == -1
    assert lib.bb200_amcl_batch_set_beam_map(None, C.byref(p), None) == -1
    assert lib.bb200_amcl_batch_set_beam_map(None, None, C.byref(g)) == -1


def test_python_exposes_the_entry_point(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    assert _capi.SIGNATURES["bb200_amcl_batch_set_beam_map"] == (C.c_int, [C.c_void_p, C.POINTER(_capi.BeamParam), C.POINTER(_capi.OccupancyGrid)])
    assert callable(bb.AmclBatch.set_beam_map)
    assert lib.bb200_abi_version() == 2
