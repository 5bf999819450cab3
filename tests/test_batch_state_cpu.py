"""State blobs without a GPU: the codec's round trip, section lengths and refusals (tests/cpp/state_blob_probe.cpp, compiled
against the library's codec source), the new entry points' declarations, exports, ctypes table and null-argument checks,
bb200_amcl_state_params and the Python wrappers' wiring."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NO_DEVICE = -1, -3
NEW = ["bb200_amcl_export_state", "bb200_amcl_create_from_state", "bb200_amcl_state_params", "bb200_amcl_batch_export_members",
       "bb200_amcl_batch_export_member", "bb200_amcl_batch_import_member", "bb200_amcl_batch_create_from_states"]


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


@pytest.fixture(scope="module")
def probe_blob(tmp_path_factory):
    out = tmp_path_factory.mktemp("state_blob_probe")  # the checkout may be read-only
    exe, blob = str(out / "probe"), str(out / "blob.bin")
    csrc = os.path.join(ROOT, "beluga_b200", "csrc")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", csrc, os.path.join(ROOT, "tests", "cpp", "state_blob_probe.cpp"),
           os.path.join(csrc, "state_blob.cpp"), "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, build.stderr[-4000:]
    run = subprocess.run([exe, blob], capture_output=True, text=True, timeout=60)
    assert run.returncode == 0 and "STATE_BLOB_PROBE_OK" in run.stdout, run.stdout + run.stderr
    with open(blob, "rb") as f:
        return f.read()


def test_codec_round_trip_sections_and_refusals(probe_blob):
    assert probe_blob[:8] == b"BB200STA"


def test_symbols_declared_exported_and_wrapped(lib):
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    with open(os.path.join(ROOT, "include", "beluga_b200.h")) as f:
        header = f.read()
    for decl in [r"int bb200_amcl_export_state\(bb200_amcl\* a, void\* out, uint64_t capacity, uint64_t\* size\);",
                 r"int bb200_amcl_create_from_state\(const void\* blob, uint64_t size, int device, bb200_amcl\*\* out\);",
                 r"int bb200_amcl_state_params\(const void\* blob, uint64_t size, bb200_amcl_param\* params, bb200_motion_param\* motion\);",
                 r"int bb200_amcl_batch_export_members\(bb200_amcl_batch\* b, const uint8_t\* present, void\* const\* out, const uint64_t\* capacity, "
                 r"uint64_t\* size\);",
                 r"int bb200_amcl_batch_export_member\(bb200_amcl_batch\* b, int member, void\* out, uint64_t capacity, uint64_t\* size\);",
                 r"int bb200_amcl_batch_import_member\(bb200_amcl_batch\* b, const void\* blob, uint64_t size, int map_id, int\* member\);",
                 r"int bb200_amcl_batch_create_from_states\(const void\* const\* blobs, const uint64_t\* sizes, int n_members, uint32_t flags, int device,\s+"
                 r"bb200_amcl_batch\*\* out\);"]:
        assert re.search(decl, header), decl
    assert re.search(r"#define BB200_ABI_VERSION 2\b", header)
    nm = subprocess.run(["nm", "-D", "--defined-only", bb_build.LIB], capture_output=True, text=True, check=True).stdout
    for name in NEW:
        assert re.search(rf"\bT {name}$", nm, re.M), name
        assert name in _capi.SIGNATURES, name
    vp, u64 = C.c_void_p, C.c_uint64
    assert _capi.SIGNATURES["bb200_amcl_batch_export_members"] == (C.c_int, [vp, C.POINTER(C.c_uint8), C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)])
    assert _capi.SIGNATURES["bb200_amcl_batch_import_member"] == (C.c_int, [vp, vp, u64, C.c_int, C.POINTER(C.c_int)])
    assert _capi.SIGNATURES["bb200_amcl_batch_create_from_states"] == (C.c_int, [C.POINTER(vp), C.POINTER(u64), C.c_int, C.c_uint32, C.c_int,
                                                                                C.POINTER(vp)])
    assert lib.bb200_abi_version() == 2


def test_null_arguments(lib, probe_blob):
    size, slot, h = C.c_uint64(5), C.c_int(-7), C.c_void_p()
    assert lib.bb200_amcl_export_state(None, None, 0, C.byref(size)) == INVALID and size.value == 5
    assert lib.bb200_amcl_create_from_state(probe_blob, len(probe_blob), 0, None) == INVALID
    assert lib.bb200_amcl_create_from_state(None, 0, 0, C.byref(h)) == INVALID and not h.value
    assert lib.bb200_amcl_batch_export_members(None, None, None, None, C.byref(size)) == INVALID
    assert lib.bb200_amcl_batch_export_member(None, 0, None, 0, C.byref(size)) == INVALID and size.value == 5
    assert lib.bb200_amcl_batch_import_member(None, probe_blob, len(probe_blob), -1, C.byref(slot)) == INVALID and slot.value == -7
    blobs, sizes = (C.c_void_p * 1)(C.cast(C.c_char_p(probe_blob), C.c_void_p)), (C.c_uint64 * 1)(len(probe_blob))
    assert lib.bb200_amcl_batch_create_from_states(None, sizes, 1, 0, 0, C.byref(h)) == INVALID
    assert lib.bb200_amcl_batch_create_from_states(blobs, sizes, 0, 0, 0, C.byref(h)) == INVALID and not h.value
    from beluga_b200 import _capi

    assert lib.bb200_amcl_state_params(probe_blob, len(probe_blob), None, C.byref(_capi.MotionParam())) == INVALID


def test_state_params_and_refusals_through_the_library(lib, probe_blob):
    import beluga_b200 as bb

    params, motion = bb.state_params(probe_blob)
    assert (params.max_particles, params.min_particles, params.resample_interval, params.seed, params.record_ancestors) == (4096, 1000, 3, 77, True)
    assert isinstance(motion, bb.OmnidirectionalDriveModelParam) and motion.strafe_noise_from_translation == 0.25
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.state_params(probe_blob[:-8])
    assert e.value.status == INVALID and "state blob: the header gives" in str(e.value)
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.state_params(b"Y" + probe_blob[1:])
    assert "wrong magic" in str(e.value)
    h = C.c_void_p()
    if bb.device_count() == 0:  # a valid blob reaches the device check; a malformed one never does
        assert lib.bb200_amcl_create_from_state(probe_blob, len(probe_blob), 0, C.byref(h)) == NO_DEVICE and not h.value
        blobs, sizes = (C.c_void_p * 1)(C.cast(C.c_char_p(probe_blob), C.c_void_p)), (C.c_uint64 * 1)(len(probe_blob))
        assert lib.bb200_amcl_batch_create_from_states(blobs, sizes, 1, 1, 0, C.byref(h)) == NO_DEVICE and not h.value
    assert lib.bb200_amcl_create_from_state(probe_blob[:100], 100, 0, C.byref(h)) == INVALID and not h.value
    assert "state blob" in lib.bb200_create_error().decode()


class FakeLib:
    """The batch entry points the state wrappers call: blobs are b"blob<slot>" padded to 120 bytes."""

    def __init__(self, occupied, blob):
        self.occupied, self.blob, self.calls = list(occupied), blob, []

    def bb200_amcl_batch_export_members(self, h, mask, out, capacity, size):
        self.calls.append(("export", out is not None))
        for m, on in enumerate(self.occupied):
            if not on or (mask is not None and not mask[m]):
                continue
            size[m] = len(self.blob)
            if out is not None:
                C.memmove(out[m], self.blob, len(self.blob))
        return 0

    def bb200_amcl_batch_import_member(self, h, blob, size, map_id, out):
        slot = self.occupied.index(False) if False in self.occupied else len(self.occupied)
        if slot == len(self.occupied):
            self.occupied.append(True)
        self.occupied[slot] = True
        self.calls.append(("import", slot, map_id, size))
        C.cast(out, C.POINTER(C.c_int))[0] = slot
        return 0

    def bb200_amcl_batch_members(self, h):
        return len(self.occupied)

    def bb200_amcl_state_params(self, blob, size, p, m):
        from beluga_b200 import _capi

        return _capi.load().bb200_amcl_state_params(blob, size, p, m)


def test_python_wiring(probe_blob):
    import beluga_b200 as bb

    b = object.__new__(bb.AmclBatch)
    b._lib = FakeLib([True, False, True], probe_blob)
    b._h = None
    b.params = [bb.AmclParams(min_particles=100, max_particles=100), None, bb.AmclParams(min_particles=100, max_particles=100)]
    b.adaptive = b.selective = False
    b._field_shapes = {}
    assert b.export_members() == [probe_blob, None, probe_blob]
    assert b.export_members(present=[0, 0, 1]) == [None, None, probe_blob]
    assert b._lib.calls[:2] == [("export", False), ("export", True)]
    assert b.import_member(probe_blob, 2) == 1 and b.params[1].max_particles == 4096
    assert b.import_member(probe_blob) == 3 and len(b.params) == 4 and b.params[3].record_ancestors
    assert b._lib.calls[-2:] == [("import", 1, 2, len(probe_blob)), ("import", 3, -1, len(probe_blob))]


def test_cpp_wrapper_declares_state_calls():
    with open(os.path.join(ROOT, "include", "beluga_b200", "amcl.hpp")) as f:
        src = f.read()
    for decl in ["std::vector<std::uint8_t> export_state() const", "static Amcl from_state(const std::vector<std::uint8_t>& blob, MotionModel motion_model",
                 "std::vector<std::uint8_t> export_member(std::size_t member) const",
                 "std::vector<std::vector<std::uint8_t>> export_members(const std::vector<bool>* present = nullptr) const",
                 "std::size_t import_member(const std::vector<std::uint8_t>& blob, int map_id = -1)",
                 "static AmclBatch from_states(const std::vector<std::vector<std::uint8_t>>& blobs"]:
        assert decl in src, decl
