"""KLD-adaptive batch members without a GPU: bb200_amcl_batch_create_adaptive accepts what bb200_amcl_create accepts for a
member (min_particles <= max_particles) and keeps the batch's other refusals, all before any device is touched; the fixed
entry point still refuses min_particles != max_particles; the new symbols are declared, exported and wrapped."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def member(**kw):
    import beluga_b200 as bb

    base = dict(min_particles=500, max_particles=2000)
    base.update(kw)
    return bb.AmclParams(**base)


def create(lib, params, adaptive=True):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    motions = [bb.DifferentialDriveModelParam() for _ in params]
    p = (_capi.AmclParam * len(params))(*[q.c() for q in params])
    m = (_capi.MotionParam * len(motions))(*[q.c_motion() for q in motions])
    h = C.c_void_p()
    fn = lib.bb200_amcl_batch_create_adaptive if adaptive else lib.bb200_amcl_batch_create
    st = fn(p, m, len(params), C.byref(h))
    if h:
        lib.bb200_amcl_batch_destroy(h)
    return st, lib.bb200_create_error().decode()


@pytest.mark.parametrize("bad,needle", [
    (dict(min_particles=2001), "min_particles <= max_particles"),
    (dict(min_particles=32768, max_particles=100), "min_particles <= max_particles"),
    (dict(selective_resampling=True), "selective"),
    (dict(shard_capacity=1000), "sharded"),
    (dict(shard_first_index=1000), "sharded"),
    (dict(min_particles=0, max_particles=0), "max_particles"),
    (dict(min_particles=500, max_particles=32769), "max_particles"),
    (dict(device=1), "one device"),
    (dict(alpha_slow=0.5, alpha_fast=0.1), "alpha_slow"),
])
def test_adaptive_rejections(lib, bad, needle):
    params = [member(), member(seed=1, min_particles=2000), member(seed=2, **bad)]
    st, message = create(lib, params)
    assert st == -1  # BB200_ERR_INVALID_ARGUMENT, with or without a device
    assert needle in message and "member 2" in message


@pytest.mark.parametrize("sizes", [(500, 2000), (1, 32768), (100, 101), (2000, 2000), (0, 1)])
def test_fixed_entry_point_still_refuses_adaptive_members(lib, sizes):
    lo, hi = sizes
    st, message = create(lib, [member(min_particles=2000, max_particles=2000), member(min_particles=lo, max_particles=hi)], adaptive=False)
    if lo == hi:
        assert st in (0, -3)  # created, or BB200_ERR_NO_DEVICE
    else:
        assert st == -1 and "fixed particle count" in message and "member 1" in message


def test_adaptive_members_pass_the_checks(lib):
    """min < max, min == max and the extremes pass validation; without a device creation then fails with
    BB200_ERR_NO_DEVICE."""
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    params = [member(), member(min_particles=1, max_particles=32768, resample_scheme=1), member(min_particles=100, max_particles=101),
              member(min_particles=2000, max_particles=2000, record_ancestors=True), member(min_particles=0, max_particles=1)]
    st, message = create(lib, params)
    assert st == -3, message
    motions = [bb.DifferentialDriveModelParam(), bb.OmnidirectionalDriveModelParam(), bb.StationaryModelParam(),
               bb.DifferentialDriveModelParam(), bb.StationaryModelParam()]
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch(motions, params, adaptive=True)
    assert e.value.status == -3
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch(motions, params)  # the fixed entry point refuses them before looking for a device
    assert e.value.status == -1 and "fixed particle count" in str(e.value)


def test_member_size_null_arguments(lib):
    from beluga_b200 import _capi

    n = C.c_uint64(7)
    assert lib.bb200_amcl_batch_member_size(None, 0, C.byref(n)) == _capi.ERR_INVALID_ARGUMENT
    assert n.value == 7
    assert lib.bb200_amcl_batch_create_adaptive(None, None, 1, None) == _capi.ERR_INVALID_ARGUMENT


def test_symbols_declared_exported_and_wrapped(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    with open(os.path.join(ROOT, "include", "beluga_b200.h")) as f:
        header = f.read()
    assert re.search(r"int bb200_amcl_batch_create_adaptive\(const bb200_amcl_param\* params, const bb200_motion_param\* motions, "
                     r"int n_members, bb200_amcl_batch\*\* out\);", header)
    assert re.search(r"int bb200_amcl_batch_member_size\(const bb200_amcl_batch\* b, int member, uint64_t\* n\);", header)
    assert re.search(r"#define BB200_ABI_VERSION 2\b", header)
    from beluga_b200 import build as bb_build

    nm = subprocess.run(["nm", "-D", "--defined-only", bb_build.LIB], capture_output=True, text=True, check=True).stdout
    for name in ("bb200_amcl_batch_create_adaptive", "bb200_amcl_batch_member_size"):
        assert re.search(rf"\bT {name}$", nm, re.M), name
    assert _capi.SIGNATURES["bb200_amcl_batch_create_adaptive"] == _capi.SIGNATURES["bb200_amcl_batch_create"]
    assert _capi.SIGNATURES["bb200_amcl_batch_member_size"] == (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)])
    assert callable(bb.AmclBatch.member_size)
    assert lib.bb200_abi_version() == 2
