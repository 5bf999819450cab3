"""Selective-resampling batch members without a GPU: bb200_amcl_batch_create_with_flags with BB200_BATCH_SELECTIVE accepts
members with selective_resampling, with BB200_BATCH_ADAPTIVE too it also accepts KLD members, unknown flag bits are
refused, and every other refusal stays, all before any device is touched; the new symbol is declared, exported and
wrapped, and AmclBatch(..., selective=True) passes the flag."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTIVE, SELECTIVE = 1, 2


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def member(**kw):
    import beluga_b200 as bb

    base = dict(min_particles=2000, max_particles=2000, selective_resampling=True)
    base.update(kw)
    return bb.AmclParams(**base)


def create(lib, params, flags):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    motions = [bb.DifferentialDriveModelParam() for _ in params]
    p = (_capi.AmclParam * len(params))(*[q.c() for q in params])
    m = (_capi.MotionParam * len(motions))(*[q.c_motion() for q in motions])
    h = C.c_void_p()
    st = lib.bb200_amcl_batch_create_with_flags(p, m, len(params), flags, C.byref(h))
    if h:
        lib.bb200_amcl_batch_destroy(h)
    return st, lib.bb200_create_error().decode()


def passes(st):
    return st in (0, -3)  # created, or BB200_ERR_NO_DEVICE: validation passed


@pytest.mark.parametrize("flags", [SELECTIVE, ADAPTIVE | SELECTIVE])
def test_selective_members_pass_the_checks(lib, flags):
    params = [member(), member(resample_interval=3, resample_scheme=1), member(selective_resampling=False, seed=3),
              member(min_particles=1, max_particles=1, recovery_probability_override=0.1)]
    st, message = create(lib, params, flags)
    assert passes(st), message


def test_selective_without_adaptive_refuses_kld_members(lib):
    st, message = create(lib, [member(), member(min_particles=500)], SELECTIVE)
    assert st == -1 and "fixed particle count" in message and "member 1" in message
    st, message = create(lib, [member(), member(min_particles=500), member(min_particles=1, max_particles=32768, selective_resampling=False)],
                         ADAPTIVE | SELECTIVE)
    assert passes(st), message


@pytest.mark.parametrize("flags", [0, ADAPTIVE])
def test_without_selective_the_flag_functions_refuse_selective_members(lib, flags):
    st, message = create(lib, [member(selective_resampling=False), member(min_particles=500 if flags else 2000)], flags)
    assert st == -1 and "selective" in message and "member 1" in message


@pytest.mark.parametrize("flags", [4, 8, 0x80000000, 0xFFFFFFFF, SELECTIVE | 4])
def test_unknown_flags(lib, flags):
    st, message = create(lib, [member()], flags)
    assert st == -1 and "flags" in message


@pytest.mark.parametrize("bad,needle", [
    (dict(min_particles=2001), "min_particles <= max_particles"),
    (dict(shard_capacity=1000), "sharded"),
    (dict(shard_first_index=1000), "sharded"),
    (dict(min_particles=0, max_particles=0), "max_particles"),
    (dict(min_particles=500, max_particles=32769), "max_particles"),
    (dict(device=1), "one device"),
    (dict(alpha_slow=0.5, alpha_fast=0.1), "alpha_slow"),
])
def test_other_refusals_stay(lib, bad, needle):
    params = [member(), member(seed=1, min_particles=1000), member(seed=2, **bad)]
    st, message = create(lib, params, ADAPTIVE | SELECTIVE)
    assert st == -1  # BB200_ERR_INVALID_ARGUMENT, with or without a device
    assert needle in message and "member 2" in message


def test_null_arguments(lib):
    assert lib.bb200_amcl_batch_create_with_flags(None, None, 1, SELECTIVE, None) == -1
    h = C.c_void_p()
    assert lib.bb200_amcl_batch_create_with_flags(None, None, 1, SELECTIVE, C.byref(h)) == -1 and not h
    st, message = create(lib, [], SELECTIVE)
    assert st == -1 and "at least one member" in message


def test_python_wiring(lib, monkeypatch):
    """AmclBatch passes adaptive and selective as the two flag bits, and refuses what the library refuses."""
    import beluga_b200 as bb
    from beluga_b200 import _capi

    assert (_capi.BATCH_ADAPTIVE, _capi.BATCH_SELECTIVE) == (ADAPTIVE, SELECTIVE)
    seen = []
    real = _capi.load()

    class Spy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if name != "bb200_amcl_batch_create_with_flags":
                return fn

            def wrapped(p, m, k, flags, out):
                seen.append(flags)
                return fn(p, m, k, flags, out)

            return wrapped

    monkeypatch.setattr(_capi, "load", lambda: Spy())
    motions = [bb.DifferentialDriveModelParam()]
    for kw, want in ((dict(), 0), (dict(adaptive=True), ADAPTIVE), (dict(selective=True), SELECTIVE),
                     (dict(adaptive=True, selective=True), ADAPTIVE | SELECTIVE)):
        try:
            b = bb.AmclBatch(motions, [member(selective_resampling=False)], **kw)
            assert b.selective == bool(kw.get("selective")) and b.adaptive == bool(kw.get("adaptive"))
        except bb.BelugaB200Error as e:
            assert e.status == -3  # no device
        assert seen[-1] == want
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch(motions, [member()])
    assert e.value.status == -1 and "selective" in str(e.value)


def test_symbols_declared_exported_and_wrapped(lib):
    from beluga_b200 import _capi

    with open(os.path.join(ROOT, "include", "beluga_b200.h")) as f:
        header = f.read()
    assert re.search(r"int bb200_amcl_batch_create_with_flags\(const bb200_amcl_param\* params, const bb200_motion_param\* motions, "
                     r"int n_members, uint32_t flags,\s+bb200_amcl_batch\*\* out\);", header)
    assert re.search(r"BB200_BATCH_ADAPTIVE = 1\b", header) and re.search(r"BB200_BATCH_SELECTIVE = 2\b", header)
    assert re.search(r"#define BB200_ABI_VERSION 2\b", header)
    from beluga_b200 import build as bb_build

    nm = subprocess.run(["nm", "-D", "--defined-only", bb_build.LIB], capture_output=True, text=True, check=True).stdout
    assert re.search(r"\bT bb200_amcl_batch_create_with_flags$", nm, re.M)
    assert _capi.SIGNATURES["bb200_amcl_batch_create_with_flags"] == (
        C.c_int, [C.POINTER(_capi.AmclParam), C.POINTER(_capi.MotionParam), C.c_int, C.c_uint32, C.POINTER(C.c_void_p)])
    assert lib.bb200_abi_version() == 2
