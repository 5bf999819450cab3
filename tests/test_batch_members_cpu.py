"""Members that join and leave a batch, without a GPU: bb200_amcl_batch_add_member, _remove_member and _member_active are
declared, exported and in the ctypes table, refuse null arguments, and AmclBatch's wrappers keep `params` per slot (None
when vacant), skip vacant slots in their per-member results and find a likelihood-field map's id through an occupied slot."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = -1
NEW = ["bb200_amcl_batch_add_member", "bb200_amcl_batch_remove_member", "bb200_amcl_batch_member_active"]


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_symbols_declared_exported_and_wrapped(lib):
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    with open(os.path.join(ROOT, "include", "beluga_b200.h")) as f:
        header = f.read()
    assert re.search(r"int bb200_amcl_batch_add_member\(bb200_amcl_batch\* b, const bb200_amcl_param\* params, const bb200_motion_param\* motion, "
                     r"int\* member\);", header)
    assert re.search(r"int bb200_amcl_batch_remove_member\(bb200_amcl_batch\* b, int member\);", header)
    assert re.search(r"int bb200_amcl_batch_member_active\(const bb200_amcl_batch\* b, int member, int\* active\);", header)
    assert re.search(r"#define BB200_ABI_VERSION 2\b", header)
    nm = subprocess.run(["nm", "-D", "--defined-only", bb_build.LIB], capture_output=True, text=True, check=True).stdout
    for name in NEW:
        assert re.search(rf"\bT {name}$", nm, re.M), name
    assert _capi.SIGNATURES["bb200_amcl_batch_add_member"] == (
        C.c_int, [C.c_void_p, C.POINTER(_capi.AmclParam), C.POINTER(_capi.MotionParam), C.POINTER(C.c_int)])
    assert _capi.SIGNATURES["bb200_amcl_batch_remove_member"] == (C.c_int, [C.c_void_p, C.c_int])
    assert _capi.SIGNATURES["bb200_amcl_batch_member_active"] == (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int)])
    assert lib.bb200_abi_version() == 2


def test_null_arguments(lib):
    import beluga_b200 as bb

    p, m, slot = bb.AmclParams().c(), bb.DifferentialDriveModelParam().c_motion(), C.c_int(-1)
    assert lib.bb200_amcl_batch_add_member(None, C.byref(p), C.byref(m), C.byref(slot)) == INVALID
    assert lib.bb200_amcl_batch_remove_member(None, 0) == INVALID
    active = C.c_int(7)
    assert lib.bb200_amcl_batch_member_active(None, 0, C.byref(active)) == INVALID and active.value == 7
    assert slot.value == -1


class FakeLib:
    """The batch entry points AmclBatch's membership wrappers call, over a list of occupied flags."""

    def __init__(self, occupied):
        self.occupied = list(occupied)
        self.calls = []

    def bb200_amcl_batch_add_member(self, h, p, m, out):
        slot = self.occupied.index(False) if False in self.occupied else len(self.occupied)
        if slot == len(self.occupied):
            self.occupied.append(True)
        self.occupied[slot] = True
        C.cast(out, C.POINTER(C.c_int))[0] = slot
        self.calls.append(("add", slot))
        return 0

    def bb200_amcl_batch_remove_member(self, h, member):
        self.occupied[member] = False
        self.calls.append(("remove", member))
        return 0

    def bb200_amcl_batch_member_active(self, h, member, out):
        C.cast(out, C.POINTER(C.c_int))[0] = int(self.occupied[member])
        return 0

    def bb200_amcl_batch_set_likelihood_field_map(self, h, p, g, prob):
        self.calls.append(("set_map",))
        return 0

    def bb200_amcl_batch_member_map(self, h, member, out):
        self.calls.append(("member_map", member))
        C.cast(out, C.POINTER(C.c_int))[0] = 5 if self.occupied[member] else -1
        return 0

    def bb200_amcl_batch_cluster_estimates(self, h, p, mask, est, cells, clusters):
        return 0

    def bb200_amcl_batch_sample_states(self, h, counts, step, mask, ptrs):
        return 0

    def bb200_amcl_batch_members(self, h):
        return len(self.occupied)


def fake_batch(occupied):
    import beluga_b200 as bb

    b = object.__new__(bb.AmclBatch)
    b._lib = FakeLib(occupied)
    b._h = None
    b.params = [bb.AmclParams(min_particles=100, max_particles=100, seed=m) if on else None for m, on in enumerate(occupied)]
    b.adaptive = b.selective = False
    b._field_shapes = {}
    return b


def test_python_wiring():
    import numpy as np

    import beluga_b200 as bb

    b = fake_batch([True, True, True])
    b.remove_member(0)
    assert b.params[0] is None and not b.member_active(0) and b.member_active(1)
    q = bb.AmclParams(min_particles=300, max_particles=300, seed=9)
    assert b.add_member(bb.StationaryModelParam(), q) == 0 and b.params[0] is q
    assert b.add_member(bb.StationaryModelParam(), q) == 3 and len(b.params) == 4 and len(b) == 4
    b.remove_member(0)
    b.remove_member(1)
    # the map id comes from the first occupied slot, not from slot 0
    b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(), bb.OccupancyGrid(np.zeros((4, 6), dtype=np.int8), 0.05))
    assert ("member_map", 2) in b._lib.calls and b._field_shapes == {5: (4, 6)}
    # vacant slots get None where present is None
    est = b.cluster_estimates()
    assert est[0] is None and est[1] is None and est[2] is not None and est[3] is not None
    samples = b.sample_states(3)
    assert samples[0] is None and samples[1] is None and samples[2].shape == (3, 4)
    est = b.cluster_estimates(present=[0, 0, 1, 0])
    assert [e is None for e in est] == [True, True, False, True]


def test_cpp_wrapper_declares_membership():
    with open(os.path.join(ROOT, "include", "beluga_b200", "amcl.hpp")) as f:
        src = f.read()
    assert "std::size_t add_member(const bb200_motion_param& motion, const AmclParams& params)" in src
    assert "void remove_member(std::size_t member)" in src
    assert "bool member_active(std::size_t member) const" in src
    assert "member_map(0)" not in src
