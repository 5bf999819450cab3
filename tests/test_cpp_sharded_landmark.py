"""The C++ landmark and bearing adaptors on shards (include/beluga_b200/models.hpp: LandmarkSensorModel2d::attach and
BearingSensorModel2d::attach on a bb200_sharded_amcl, amcl.hpp: ShardedAmcl::update with a landmark token): compiles with and
without the Sophus conversions; run on a machine without a device it reports BB200_ERR_NO_DEVICE, on the GPU every step of 2
and 4 shards equals a beluga_b200::Amcl with the same parameters and seed, byte for byte."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("cpp_sharded_landmark"))


def build_exe(build_dir: str, with_sophus_stub: bool = False) -> str:
    from beluga_b200 import build as bb_build

    bb_build.build()
    lib_dir = os.path.join(ROOT, "beluga_b200")
    exe = os.path.join(build_dir, "test_sharded_landmark_adaptor" + ("_sophus" if with_sophus_stub else ""))
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_sharded_landmark_adaptor.cpp"), "-o", exe, "-L", lib_dir, "-lbeluga_b200",
           f"-Wl,-rpath,{lib_dir}"]
    if with_sophus_stub:
        cmd[1:1] = ["-DBELUGA_B200_WITH_SOPHUS", "-I", os.path.join(ROOT, "tests", "cpp", "stubs")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return exe


def test_sharded_landmark_adaptor_compiles_with_sophus_conversions(build_dir):
    build_exe(build_dir, with_sophus_stub=True)


def test_sharded_landmark_adaptor_without_device(build_dir):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    out = subprocess.run([build_exe(build_dir)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "SHARDED_LANDMARK_ADAPTOR_NO_DEVICE" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("with_sophus_stub", [False, True])
def test_sharded_landmark_adaptor_runs(build_dir, with_sophus_stub):
    out = subprocess.run([build_exe(build_dir, with_sophus_stub)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "SHARDED_LANDMARK_ADAPTOR_OK" in out.stdout, out.stdout + out.stderr
