"""bb200_amcl_batch_cluster_estimates without a GPU: a null handle or a null argument is refused with BB200_ERR_INVALID_ARGUMENT
before anything else is looked at, and the ctypes table carries the entry point."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_null_handle_and_null_arguments(lib):
    from beluga_b200 import _capi

    p = _capi.ClusterParam(0.2, 0.524, 0.9)
    out = (_capi.Estimate * 4)()
    cells, clusters = (C.c_uint32 * 4)(), (C.c_uint32 * 4)()
    assert lib.bb200_amcl_batch_cluster_estimates(None, C.byref(p), None, out, cells, clusters) == -1
    assert lib.bb200_amcl_batch_cluster_estimates(None, None, None, None, None, None) == -1
    assert lib.bb200_amcl_batch_cluster_estimates(None, C.byref(p), None, None, None, None) == -1
    assert lib.bb200_amcl_batch_cluster_estimates(None, None, None, out, None, None) == -1
    assert lib.bb200_amcl_batch_last_error(None) == b"null batch"
