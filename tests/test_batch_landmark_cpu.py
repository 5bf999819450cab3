"""Landmark maps and detections in a batch, without a GPU: the new entry points are exported, declared in
include/beluga_b200.h and carried by the ctypes table and AmclBatch; BB200_MEASUREMENT_LANDMARKS is 4 while
bb200_measurement and the ABI version stay as they were; null handles and null arguments are refused with
BB200_ERR_INVALID_ARGUMENT before anything else is looked at; and every field the batch kernels read keeps its offset in
BatchStepArgs and BatchMap (the new fields are appended)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "beluga_b200", "csrc")
INVALID = -1

NEW = {
    "bb200_amcl_batch_set_landmark_map": ("LandmarkParam", "LandmarkMap"),
    "bb200_amcl_batch_set_bearing_map": ("BearingParam", "LandmarkMap"),
    "bb200_amcl_batch_add_landmark_map": ("LandmarkParam", "LandmarkMap", "int*"),
    "bb200_amcl_batch_add_bearing_map": ("BearingParam", "LandmarkMap", "int*"),
}


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_symbols_argtypes_and_declarations(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    header = open(os.path.join(ROOT, "include", "beluga_b200.h")).read()
    P = C.POINTER
    for name, args in NEW.items():
        assert hasattr(lib, name) and re.search(rf"\bint {name}\(", header), name
        want = [C.c_void_p] + [P(C.c_int) if a == "int*" else P(getattr(_capi, a)) for a in args]
        assert _capi.SIGNATURES[name] == (C.c_int, want), name
    assert _capi.SIGNATURES["bb200_amcl_batch_set_detections"] == (C.c_int, [C.c_void_p, P(P(_capi.Landmark)), P(C.c_uint64), P(C.c_uint8)])
    assert re.search(r"\bint bb200_amcl_batch_set_detections\(bb200_amcl_batch\* b, const bb200_landmark_detection\* const\* detections, "
                     r"const uint64_t\* n, const uint8_t\* present\);", header)
    for method in ("set_landmark_map", "set_bearing_map", "add_landmark_map", "add_bearing_map"):
        assert callable(getattr(bb.AmclBatch, method)), method
    d = bb.Detections(np.zeros((2, 3)), np.zeros(2, dtype=np.uint32))
    assert d.positions.shape == (2, 3)


def test_measurement_kind_and_layout_unchanged(lib):
    from beluga_b200 import _capi

    header = open(os.path.join(ROOT, "include", "beluga_b200.h")).read()
    assert re.search(r"BB200_MEASUREMENT_LANDMARKS = 4\b", header)
    assert _capi.MEASUREMENT_LANDMARKS == 4
    assert [f[0] for f in _capi.Measurement._fields_] == ["kind", "points_xy", "n_points", "scan", "cloud"]
    assert C.sizeof(_capi.Measurement) == 40
    assert lib.bb200_abi_version() == 2


def test_null_handle_and_null_arguments(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    lp, bp = bb.LandmarkModelParam().c(), bb.BearingModelParam().c()
    lmap = bb.LandmarkMap(np.zeros((2, 3)), np.zeros(2, dtype=np.uint32))
    m = lmap.c()
    mid = C.c_int(-1)
    for set_fn, p in ((lib.bb200_amcl_batch_set_landmark_map, lp), (lib.bb200_amcl_batch_set_bearing_map, bp)):
        assert set_fn(None, C.byref(p), C.byref(m)) == INVALID
        assert set_fn(None, None, None) == INVALID
    for add_fn, p in ((lib.bb200_amcl_batch_add_landmark_map, lp), (lib.bb200_amcl_batch_add_bearing_map, bp)):
        assert add_fn(None, C.byref(p), C.byref(m), C.byref(mid)) == INVALID
        assert add_fn(None, C.byref(p), C.byref(m), None) == INVALID
    arr = (_capi.Landmark * 1)()
    ptrs = (C.POINTER(_capi.Landmark) * 1)(arr)
    n = (C.c_uint64 * 1)(1)
    assert lib.bb200_amcl_batch_set_detections(None, ptrs, n, None) == INVALID
    assert lib.bb200_amcl_batch_set_detections(None, ptrs, None, None) == INVALID
    assert mid.value == -1


def test_batch_args_keep_their_offsets(tmp_path):
    """Host-only probe: every BatchStepArgs and BatchMap field the grid kernels read sits where it sat before the landmark
    fields were appended (the parameter block grew from 640 bytes, the map entry from 416)."""
    from beluga_b200 import build as bb_build

    cuda = os.path.dirname(os.path.dirname(os.path.realpath(shutil.which(bb_build.nvcc()))))
    exe = str(tmp_path / "batch_args_probe")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O0", "-Wall", "-Wno-unknown-pragmas", "-I", CSRC, "-I", os.path.join(cuda, "include"),
           os.path.join(ROOT, "tests", "cpp", "batch_args_probe.cpp"), "-o", exe]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-4000:]
    run = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert run.returncode == 0, run.stderr
    got = dict(line.split() for line in run.stdout.strip().split("\n"))
    want = ("BatchStepArgs.members 0 BatchStepArgs.first 8 BatchStepArgs.n_members 16 BatchStepArgs.ctas 20 BatchStepArgs.max_points 44 "
            "BatchStepArgs.states 48 BatchStepArgs.weights 64 BatchStepArgs.cdf 72 BatchStepArgs.ancestors 80 BatchStepArgs.tile_state 88 "
            "BatchStepArgs.scalars 96 BatchStepArgs.partials 104 BatchStepArgs.points 112 BatchStepArgs.field 128 BatchStepArgs.free_cells 288 "
            "BatchStepArgs.n_free 296 BatchStepArgs.grid_width 304 BatchStepArgs.grid_resolution 312 BatchStepArgs.grid_origin 320 "
            "BatchStepArgs.summary 352 BatchStepArgs.members_done 360 BatchStepArgs.ticket 368 BatchStepArgs.seq 376 BatchStepArgs.forms 380 "
            "BatchStepArgs.occupancy 384 BatchStepArgs.beam 480 BatchStepArgs.hits 552 BatchStepArgs.maps 560 BatchStepArgs.kld 568 "
            "BatchStepArgs.hashes 576 BatchStepArgs.keys 584 BatchStepArgs.vals 592 BatchStepArgs.post_ctas 600 BatchStepArgs.ess_ctas 608 "
            "BatchStepArgs.weigh_ctas 612 BatchStepArgs.factors 616 BatchMap.field 0 BatchMap.occupancy 160 BatchMap.beam 256 "
            "BatchMap.free_cells 328 BatchMap.n_free 336 BatchMap.grid_width 344 BatchMap.grid_resolution 352 BatchMap.grid_origin 384 "
            "BatchMember.hit_stride 184 sizeof.BatchMember 192").split()
    want = dict(zip(want[::2], want[1::2]))
    assert {k: got[k] for k in want} == want
    assert 640 < int(got["sizeof.BatchStepArgs"]) <= 1024
    assert int(got["sizeof.BatchMap"]) > 416
