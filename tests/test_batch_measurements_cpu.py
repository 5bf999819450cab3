"""bb200_amcl_batch_update_measurements without a GPU: a null handle or a null required argument is refused with
BB200_ERR_INVALID_ARGUMENT; the ctypes table and AmclBatch carry the entry point; AmclBatch refuses a measurement list of
the wrong length and the wrong kinds before reaching the library; a batch cannot be created without a device
(BB200_ERR_NO_DEVICE); and the host half of a scan's conversion that the batch shares with bb200_scan_to_points
(csrc/measurement_host.hpp: the kept indices and the beam directions) gives bb200_scan_to_points's points."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from beluga_b200 import _capi
    from beluga_b200 import build as bb_build

    bb_build.build()
    return _capi.load()


def test_null_handle_and_null_arguments(lib):
    from beluga_b200 import _capi

    k = 2
    poses = np.zeros((k, 4))
    table = (_capi.Measurement * k)()
    res = (_capi.UpdateResult * k)()
    res[0].updated = 7
    p = poses.ctypes.data_as(C.POINTER(C.c_double))
    assert lib.bb200_amcl_batch_update_measurements(None, p, table, None, res) == _capi.ERR_INVALID_ARGUMENT
    assert lib.bb200_amcl_batch_update_measurements(None, None, table, None, res) == _capi.ERR_INVALID_ARGUMENT
    assert lib.bb200_amcl_batch_update_measurements(None, p, None, None, res) == _capi.ERR_INVALID_ARGUMENT
    assert lib.bb200_amcl_batch_update_measurements(None, p, table, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert res[0].updated == 7


def test_python_exposes_the_entry_point(lib):
    import beluga_b200 as bb
    from beluga_b200 import _capi

    assert _capi.SIGNATURES["bb200_amcl_batch_update_measurements"] == (
        C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(_capi.Measurement), C.POINTER(C.c_uint8), C.POINTER(_capi.UpdateResult)])
    assert [f for f, _ in _capi.Measurement._fields_] == ["kind", "points_xy", "n_points", "scan", "cloud"]
    assert C.sizeof(_capi.Measurement) == 40
    for name in ("update_measurements", "update_scans", "update_point_clouds"):
        assert callable(getattr(bb.AmclBatch, name)), name
    assert lib.bb200_abi_version() == 2


class _NoCalls:
    def __getattr__(self, name):
        raise AssertionError(f"{name} called despite a malformed argument")


def test_lengths_and_kinds_are_checked_before_the_library(lib):
    import beluga_b200 as bb

    b = bb.AmclBatch.__new__(bb.AmclBatch)  # no device here: the checks under test run before any library call
    b._lib = _NoCalls()
    b._h = None
    b.params = [bb.AmclParams(min_particles=10, max_particles=10) for _ in range(3)]
    scan = bb.LaserScan(np.ones(10, dtype=np.float32), -1.0, 0.1)
    with pytest.raises(ValueError, match="one measurement per member"):
        b.update_measurements(np.zeros((3, 4)), [scan, scan])
    with pytest.raises(ValueError, match="presence flag"):
        b.update_measurements(np.zeros((3, 4)), [scan] * 3, present=[True])
    with pytest.raises(TypeError, match="LaserScan"):
        b.update_scans(np.zeros((3, 4)), [scan, np.zeros((0, 2)), scan])
    with pytest.raises(TypeError, match="PointCloud"):
        b.update_point_clouds(np.zeros((3, 4)), [scan] * 3)


def test_batch_needs_a_device(lib):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.AmclBatch([bb.StationaryModelParam()], [bb.AmclParams(min_particles=10, max_particles=10)])
    assert e.value.status == -3


PROBE = r"""
#include "measurement_host.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>
// Every scan below through the shared host half (kept indices, directions) plus the range filter and origin the batch
// kernel applies, against bb200_scan_to_points and bb200_take_evenly_indices; prints the cases checked.
int main() {
  int cases = 0;
  const double origin[12] = {0.8, -0.6, 0.01, 0.3, 0.6, 0.8, -0.02, -1.7, 0.0, 0.0, 1.0, 0.4};
  for (uint64_t n : std::vector<uint64_t>{0, 1, 2, 3, 181, 1080, 4001}) {
    std::vector<float> ranges(n);
    for (uint64_t i = 0; i < n; ++i) ranges[i] = 0.1f + 0.37f * static_cast<float>(i % 97);
    if (n > 5) ranges[3] = NAN, ranges[4] = INFINITY, ranges[5] = -INFINITY;
    for (uint64_t max_beams : std::vector<uint64_t>{0, 1, 2, n > 0 ? n - 1 : 0, n, n + 3, 100}) {
      for (const double* o : {static_cast<const double*>(nullptr), origin}) {
        const bb200_laser_scan scan{ranges.data(), n, -3.1f, 0.0058f, 0.2, 30.0, max_beams, o};
        std::vector<double> want(2 * (n + 1));
        uint64_t n_want = 0;
        if (bb200_scan_to_points(&scan, want.data(), n + 1, &n_want) != BB200_OK) return 1;
        const uint64_t kept = bb200::scan_beam_count(scan);
        std::vector<uint64_t> idx(n + 1);
        uint64_t n_idx = 0;
        if (bb200_take_evenly_indices(n, max_beams == 0 ? n : max_beams, idx.data(), n + 1, &n_idx) != BB200_OK || n_idx != kept) return 2;
        std::vector<double> got;
        for (uint64_t pos = 0; pos < kept; ++pos) {
          const bb200::ScanBeam beam = bb200::scan_beam(scan, pos);
          if (beam.index != idx[pos]) return 3;
          const double r = ranges[beam.index];
          if (!bb200::scan_range_kept(r, scan)) continue;
          const double x = r * beam.c, y = r * beam.s;
          got.push_back(o != nullptr ? (o[0] * x + o[1] * y) + o[3] : x);
          got.push_back(o != nullptr ? (o[4] * x + o[5] * y) + o[7] : y);
        }
        if (got.size() != 2 * n_want || (n_want > 0 && std::memcmp(got.data(), want.data(), got.size() * sizeof(double)) != 0)) return 4;
        ++cases;
      }
    }
  }
  std::printf("%d\n", cases);
  return 0;
}
"""


def test_shared_scan_host_half_matches_scan_to_points(lib, tmp_path):
    src = tmp_path / "scan_probe.cpp"
    src.write_text(PROBE)
    exe = str(tmp_path / "scan_probe")
    lib_dir = os.path.join(ROOT, "beluga_b200")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror", "-I", os.path.join(lib_dir, "csrc"), str(src), "-o", exe,
           "-L", lib_dir, "-lbeluga_b200", f"-Wl,-rpath,{lib_dir}"]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    run = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0 and int(run.stdout) == 7 * 7 * 2, (run.returncode, run.stdout, run.stderr)
