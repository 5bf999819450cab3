"""Batched particle-cloud publication without a GPU: bb200_amcl_batch_particle_histograms and bb200_amcl_batch_sample_states
refuse a null handle or a null required argument with BB200_ERR_INVALID_ARGUMENT and write nothing; the ctypes table and
AmclBatch carry the entry points; AmclBatch refuses a presence mask or a count list of the wrong length, and negative
counts, before reaching the library; and the ABI version stays 2."""
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
    from beluga_b200 import _capi

    k = 3
    bufs = [(_capi.ClusterCell * 4)() for _ in range(k)]
    bins = (C.POINTER(_capi.ClusterCell) * k)(*[C.cast(b, C.POINTER(_capi.ClusterCell)) for b in bufs])
    capacity = (C.c_uint64 * k)(4, 4, 4)
    n_bins = (C.c_uint64 * k)(*([77] * k))
    top = (C.c_double * k)(*([-1.0] * k))
    mask = (C.c_uint8 * k)(1, 0, 1)
    assert lib.bb200_amcl_batch_particle_histograms(None, 1e-3, 1e-3, mask, bins, capacity, n_bins, top) == -1
    assert lib.bb200_amcl_batch_particle_histograms(None, 1e-3, 1e-3, None, None, None, None, None) == -1
    assert lib.bb200_amcl_batch_particle_histograms(None, 0.0, -1.0, None, bins, capacity, n_bins, top) == -1
    assert list(n_bins) == [77] * k and list(top) == [-1.0] * k

    outs = [np.full((2, 4), 5.0) for _ in range(k)]
    ptrs = (C.POINTER(C.c_double) * k)(*[o.ctypes.data_as(C.POINTER(C.c_double)) for o in outs])
    counts = (C.c_uint64 * k)(2, 2, 2)
    assert lib.bb200_amcl_batch_sample_states(None, counts, 0, mask, ptrs) == -1
    assert lib.bb200_amcl_batch_sample_states(None, None, 0, None, ptrs) == -1
    assert lib.bb200_amcl_batch_sample_states(None, counts, 0, None, None) == -1
    assert lib.bb200_amcl_batch_sample_states(None, None, 0, None, None) == -1
    assert all(np.all(o == 5.0) for o in outs)
    assert lib.bb200_amcl_batch_last_error(None) == b"null batch"


def test_python_exposes_the_entry_points(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    vp, u64p, u8p = C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
    assert _capi.SIGNATURES["bb200_amcl_batch_particle_histograms"] == (
        C.c_int, [vp, C.c_double, C.c_double, u8p, C.POINTER(C.POINTER(_capi.ClusterCell)), u64p, u64p, C.POINTER(C.c_double)])
    assert _capi.SIGNATURES["bb200_amcl_batch_sample_states"] == (C.c_int, [vp, u64p, C.c_uint32, u8p, C.POINTER(C.POINTER(C.c_double))])
    for name in ("particle_histograms", "sample_states"):
        assert callable(getattr(bb.AmclBatch, name)), name
    assert bb._CELL_DTYPE.itemsize == C.sizeof(_capi.ClusterCell)
    assert lib.bb200_abi_version() == 2


class _NoCalls:
    """A library stand-in that fails the test if AmclBatch reaches it."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} called despite a malformed argument")


def _unbound_batch(bb, k):
    b = bb.AmclBatch.__new__(bb.AmclBatch)  # no device here: the checks under test run before any library call
    b._lib = _NoCalls()
    b._h = None
    b.params = [bb.AmclParams(min_particles=10, max_particles=10) for _ in range(k)]
    return b


def test_mask_and_count_lengths_are_checked(lib):
    import beluga_b200 as bb

    b = _unbound_batch(bb, 3)
    with pytest.raises(ValueError, match="presence flag"):
        b.particle_histograms(present=[True, False])
    with pytest.raises(ValueError, match="presence flag"):
        b.sample_states(1, present=[True] * 4)
    with pytest.raises(ValueError, match="sample count"):
        b.sample_states([1, 2])
    with pytest.raises(ValueError, match="negative"):
        b.sample_states([1, -2, 3])
