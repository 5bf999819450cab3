"""The CPU model tests restate pieces of csrc/kernels.cuh in Python.  This test compiles a host-only probe against the real
header (tests/cpp/schedule_probe.cu; nvcc, no GPU needed, no CUDA call) and checks that the restatements compute what the
code the kernels are built from computes: the pose-bin grid of the execution schedule and the bordered tile layout."""
import os
import shutil
import subprocess

import pytest

from test_fixed_point_lookup_model import bordered_index, kernel_index
from test_schedule_model import MAX_BINS, schedule_from_moments

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = [
    (0.45, 0.87, 30.0, 40.0, 0.25, 0.30, 1e6, 21.0, 0.025),
    (0.45, 0.87, 30.0, 40.0, 0.25, 0.30, 1.25e7, 21.0, 0.025),
    (1.0, 0.0, 3.0, 4.0, 0.0, 0.0, 1e4, 10.0, 0.025),
    (0.0, 0.0, 0.0, 0.0, 1.0, 1.0, 1e4, 10.0, 0.025),
    (-0.2, 0.1, -5.0, 7.5, 4.0, 0.01, 32769.0, 3.0, 0.05),
    (0.486, -0.648, 12.5, -3.0, 0.04, 2.25, 2.5e5, 8.0, 0.05),
]


@pytest.fixture(scope="module")
def probe_lines(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    exe = str(tmp_path_factory.mktemp("schedule_probe") / "schedule_probe")  # the checkout may be read-only
    cmd = [nvcc, "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "beluga_b200", "csrc"), "-o", exe,
           os.path.join(ROOT, "tests", "cpp", "schedule_probe.cu")]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-3000:]
    run = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert run.returncode == 0
    return run.stdout.splitlines()


def test_schedule_grid_matches_the_header(probe_lines):
    grids = [line.split()[1:] for line in probe_lines if line.startswith("grid ")]
    assert len(grids) == len(CASES)  # keep CASES in step with tests/cpp/schedule_probe.cu
    assert int([line for line in probe_lines if line.startswith("max_bins ")][0].split()[1]) == MAX_BINS
    for case, got in zip(CASES, grids):
        g = schedule_from_moments(*case)
        nt, nx, ny, n_bins = (int(v) for v in got[:4])
        assert (nt, nx, ny, n_bins) == (g["nt"], g["nx"], g["ny"], g["n_bins"]), case
        for a, b in zip((float(v) for v in got[4:7]), (g["c0"], g["s0"], g["half_u"])):
            assert a == pytest.approx(b, rel=1e-12, abs=1e-12), case
        for a, b in zip((float(v) for v in got[7:10]), (g["kt"], g["kx"], g["ky"])):
            assert a == pytest.approx(float(b), rel=1e-6), case


def test_bordered_index_matches_the_header(probe_lines):
    rows = [tuple(int(v) for v in line.split()[1:]) for line in probe_lines if line.startswith("index ")]
    assert len(rows) == sum(9 * (4 << kx) for kx in range(4))
    for kx, px, py, idx in rows:
        assert bordered_index(px, py, kx) == idx
        assert kernel_index(4 * px + 3, py, kx) == idx  # what the kernel's three integer operations make of the same cell


def test_counter_rng_and_spatial_hash_of_the_product_header(probe_lines, orc):
    """se2_math.cuh compiled for the host: Philox4x32-10 known answers (Random123's kat_vectors), and the spatial hash of 64
    poses against the oracle's restatement of algorithm/spatial_hash.hpp:45-94,190-193."""
    import numpy as np

    philox = [line.split()[1:] for line in probe_lines if line.startswith("philox ")]
    assert philox == [["6627e8d5", "e169c58d", "bc57ac4c", "9b00dbd8"], ["408f276d", "41c83b0e", "a20bc7c6", "6d5451fd"],
                      ["d16cfe09", "94fdcceb", "5001e420", "24126ea1"]]
    rows = [line.split()[1:] for line in probe_lines if line.startswith("hash ")]
    assert len(rows) == 64
    for r in rows:
        state = np.array([float(v) for v in r[:4]])
        assert orc.spatial_hash(state, 0.5, 0.5, 0.17453292519943295) == int(r[4])
        assert orc.spatial_hash(state, 0.05, 0.1, 0.01) == int(r[5])
        z0, z1 = float(r[6]), float(r[7])
        assert np.isfinite(z0) and np.isfinite(z1) and abs(z0) < 9.0 and abs(z1) < 9.0
    z = np.array([[float(r[6]), float(r[7])] for r in rows]).reshape(-1)
    assert abs(z.mean()) < 0.35 and 0.7 < z.std() < 1.3  # 128 standard normals
