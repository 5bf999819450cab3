"""bb200_amcl_batch_update_clustered without a GPU.

The order-defining half of the device cluster selection (csrc/cluster_select.cuh) is compiled for the host by
tests/cpp/cluster_select_probe.cpp and checked against the real containers it restates: the iteration order of
std::unordered_map after reserve(n / 5) for every distinct initial bucket count, on both sides of every rehash threshold;
the whole selection against select_cluster (bb200_cluster_select_host's code) and the oracle's clusterizer on thousands of
particle sets whose capped cells tie; and the fallback predicate's margin for headings at an angular bucket edge.  The C
symbol, the ctypes table, the argument checks and the Python wiring are checked too."""
import ctypes as C
import os
import re
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


@pytest.fixture(scope="module")
def probe(lib, tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("cluster_select_probe") / "probe")  # the checkout may be read-only
    lib_dir = os.path.join(ROOT, "beluga_b200")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror", "-Wno-unknown-pragmas", "-I", os.path.join(lib_dir, "csrc"),
           "-I", os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "cpp", "cluster_select_probe.cpp"), "-o", exe, "-L", lib_dir,
           "-lbeluga_b200", f"-Wl,-rpath,{lib_dir}"]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-4000:]
    run = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-2000:]
    return {line.split()[0]: [int(v) for v in line.split()[1:]] for line in run.stdout.splitlines()}


def test_every_reserve_starts_its_schedule(probe):
    wants, mismatches = probe["reserve"]
    assert wants == 32768 // 5 + 1 and mismatches == 0


def test_map_order_matches_unordered_map_across_rehashes(probe):
    cases, crossed, mismatches = probe["map"]
    assert cases > 500 and crossed > 100
    assert mismatches == 0


def test_selection_matches_select_cluster_and_the_oracle(probe):
    cases, tied, mismatches, oracle_mismatches = probe["select"]
    assert cases == 3000 and tied > 1000
    assert mismatches == 0 and oracle_mismatches == 0


def test_headings_the_predicate_passes_keep_their_bucket(probe):
    checked, flagged, violations = probe["edge"]
    assert checked > 100000 and flagged > 10000
    assert violations == 0


def test_symbol_header_and_ctypes(lib):
    from beluga_b200 import _capi

    header = open(os.path.join(ROOT, "include", "beluga_b200.h")).read()
    assert re.search(r"int bb200_amcl_batch_update_clustered\(bb200_amcl_batch\* b, const double\* control_poses, const bb200_measurement\* measurements,"
                     r"\s+const uint8_t\* present, const bb200_cluster_param\* p, bb200_update_result\* out,\s+bb200_estimate\* clustered, uint32_t\* n_cells,"
                     r" uint32_t\* n_clusters\);", header)
    assert _capi.SIGNATURES["bb200_amcl_batch_update_clustered"] == (
        C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(_capi.Measurement), C.POINTER(C.c_uint8), C.POINTER(_capi.ClusterParam),
                  C.POINTER(_capi.UpdateResult), C.POINTER(_capi.Estimate), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)])
    assert lib.bb200_abi_version() == 2


def test_null_handle_and_null_arguments(lib):
    from beluga_b200 import _capi

    k = 2
    poses = np.zeros((k, 4))
    p = poses.ctypes.data_as(C.POINTER(C.c_double))
    table = (_capi.Measurement * k)()
    param = _capi.ClusterParam(0.2, 0.524, 0.9)
    res = (_capi.UpdateResult * k)()
    est = (_capi.Estimate * k)()
    res[0].updated = 7
    f = lib.bb200_amcl_batch_update_clustered
    assert f(None, p, table, None, C.byref(param), res, est, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert f(None, None, table, None, C.byref(param), res, est, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert f(None, p, None, None, C.byref(param), res, est, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert f(None, p, table, None, None, res, est, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert f(None, p, table, None, C.byref(param), None, est, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert f(None, p, table, None, C.byref(param), res, None, None, None) == _capi.ERR_INVALID_ARGUMENT
    assert res[0].updated == 7


class _NoCalls:
    def __getattr__(self, name):
        raise AssertionError(f"{name} called despite a malformed argument")


def test_python_wiring_checks_lengths_before_the_library(lib):
    import beluga_b200 as bb

    assert callable(bb.AmclBatch.update_clustered)
    b = bb.AmclBatch.__new__(bb.AmclBatch)  # no device here: the checks under test run before any library call
    b._lib = _NoCalls()
    b._h = None
    b.params = [bb.AmclParams(min_particles=10, max_particles=10) for _ in range(3)]
    pts = np.zeros((4, 2))
    with pytest.raises(ValueError, match="one measurement per member"):
        b.update_clustered(np.zeros((3, 4)), [pts, pts])
    with pytest.raises(ValueError, match="presence flag"):
        b.update_clustered(np.zeros((3, 4)), [pts] * 3, present=[True])


def test_python_passes_the_parameters(lib):
    """update_clustered hands the library one cluster parameter block and K-entry outputs, and maps updated members only."""
    import beluga_b200 as bb
    from beluga_b200 import _capi

    seen = {}

    class _Fake:
        def bb200_amcl_batch_update_clustered(self, h, poses, table, mask, param, res, est, cells, clusters):
            p = C.cast(param, C.POINTER(_capi.ClusterParam)).contents
            seen["param"] = (p.linear_hash_resolution, p.angular_hash_resolution, p.weight_cap_percentile)
            seen["mask"] = None if mask is None else list(mask)
            res[1].updated = 1
            est[1].mean[0] = 1.0
            cells[1], clusters[1] = 5, 2
            return 0

    b = bb.AmclBatch.__new__(bb.AmclBatch)
    b._lib = _Fake()
    b._h = None
    b.params = [bb.AmclParams(min_particles=10, max_particles=10) for _ in range(3)]
    results, ests = b.update_clustered(np.zeros((3, 4)), [np.zeros((2, 2))] * 3, present=[True, True, False], linear=0.5, angular=0.25,
                                       percentile=0.75, with_counts=True)
    assert seen == {"param": (0.5, 0.25, 0.75), "mask": [1, 1, 0]}
    assert len(results) == 3 and ests[0] is None and ests[2] is None
    mean, cov, cells, clusters = ests[1]
    assert mean[0] == 1.0 and cov.shape == (3, 3) and (cells, clusters) == (5, 2)
