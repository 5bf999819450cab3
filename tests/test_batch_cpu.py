"""The batch of filters without a GPU: every configuration a batch rejects is refused before any device is touched, and a
valid one fails loudly for want of a device instead of computing on the host."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def member(**kw):
    import beluga_b200 as bb

    base = dict(min_particles=2000, max_particles=2000)
    base.update(kw)
    return bb.AmclParams(**base)


def create(lib, params, motions=None, n=None):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    motions = motions or [bb.DifferentialDriveModelParam() for _ in params]
    k = len(params) if n is None else n
    p = (_capi.AmclParam * max(len(params), 1))(*[q.c() for q in params])
    m = (_capi.MotionParam * max(len(motions), 1))(*[q.c_motion() for q in motions])
    h = C.c_void_p()
    st = lib.bb200_amcl_batch_create(p, m, k, C.byref(h))
    if h:
        lib.bb200_amcl_batch_destroy(h)
    return st, lib.bb200_create_error().decode()


@pytest.mark.parametrize("bad,needle", [
    (dict(min_particles=500), "fixed particle count"),  # KLD
    (dict(min_particles=3000), "fixed particle count"),
    (dict(selective_resampling=True), "selective"),
    (dict(shard_capacity=1000), "sharded"),
    (dict(shard_first_index=1000), "sharded"),
    (dict(min_particles=0, max_particles=0), "max_particles"),
    (dict(min_particles=32769, max_particles=32769), "max_particles"),
    (dict(device=1), "one device"),
    (dict(alpha_slow=0.5, alpha_fast=0.1), "alpha_slow"),
])
def test_rejected_configurations(lib, bad, needle):
    params = [member(), member(seed=1), member(seed=2, **bad)]
    st, message = create(lib, params)
    assert st == -1  # BB200_ERR_INVALID_ARGUMENT, with or without a device
    assert needle in message and "member 2" in message


def test_no_members_and_null_arguments(lib):
    st, _ = create(lib, [member()], n=0)
    assert st == -1
    assert lib.bb200_amcl_batch_create(None, None, 1, None) == -1
    assert lib.bb200_amcl_batch_update(None, None, None, None, None, None) == -1
    assert lib.bb200_amcl_batch_members(None) == 0
    assert lib.bb200_amcl_batch_launch_count(None) == 0
    assert lib.bb200_amcl_batch_last_error(None) == b"null batch"


def test_unknown_motion_model(lib):
    import beluga_b200 as bb

    class Bad(bb.StationaryModelParam):
        def c_motion(self):
            m = super().c_motion()
            m.model = 7
            return m

    st, message = create(lib, [member(), member()], motions=[bb.StationaryModelParam(), Bad()])
    assert st == -1 and "motion model" in message


def test_largest_member_is_accepted_by_the_checks(lib):
    """32768 particles and a mix of schemes, motions and policies pass validation; without a device creation then fails
    with BB200_ERR_NO_DEVICE."""
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    params = [member(min_particles=32768, max_particles=32768), member(resample_interval=3, resample_scheme=1),
              member(recovery_probability_override=0.1, record_ancestors=True)]
    motions = [bb.DifferentialDriveModelParam(), bb.OmnidirectionalDriveModelParam(), bb.StationaryModelParam()]
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch(motions, params)
    assert e.value.status == -3  # BB200_ERR_NO_DEVICE
