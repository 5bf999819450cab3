"""TEST INFRASTRUCTURE ONLY -- the CPU oracle's Ray2d::cast with raw {cos, sin} bearings (tests/cpp/raycast_oracle.cpp), built
with the oracle's compiler flags into a temporary directory, since the checkout may be read-only."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        out_dir = tempfile.mkdtemp(prefix="bb200_raycast_oracle_")
        atexit.register(shutil.rmtree, out_dir, True)
        so = os.path.join(out_dir, "libraycast_oracle.so")
        # -ffp-contract=off as oracle/Makefile: the far end and the distance round after every multiply, as the reference's do
        subprocess.run(["/usr/bin/g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror",
                        os.path.join(ROOT, "tests", "cpp", "raycast_oracle.cpp"), "-o", so], check=True)
        _lib = C.CDLL(so)
        _lib.orc_raycast_raw.restype = None
    return _lib


def cast_rays(cells, resolution: float, origin, poses, bearings, max_range: float) -> np.ndarray:
    """Ray2d::cast of every pose (n, 4) [cos, sin, x, y] along every bearing (m, 2) [cos, sin] -> (n, m), inf for a miss."""
    c = np.ascontiguousarray(cells, dtype=np.int8)
    o = np.ascontiguousarray(origin, dtype=np.float64)
    p = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 4)
    b = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 2)
    out = np.zeros((len(p), len(b)))
    d = C.POINTER(C.c_double)
    lib().orc_raycast_raw(c.ctypes.data_as(C.POINTER(C.c_int8)), c.shape[1], c.shape[0], C.c_double(resolution), o.ctypes.data_as(d),
                          p.ctypes.data_as(d), C.c_uint64(len(p)), b.ctypes.data_as(d), C.c_uint64(len(b)), C.c_double(max_range),
                          out.ctypes.data_as(d))
    return out
