"""The point-cloud input of the header-only C++ adaptors (beluga_b200::PointCloudView, point_cloud_points, the
Amcl::update(control, cloud) overloads): compiled with and without the Sophus stub headers; the host-side conversion runs
on the CPU, the filter updates on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    """Executables go to a temporary directory: the checkout may be read-only."""
    return str(tmp_path_factory.mktemp("cpp_point_cloud"))


def build_exe(build_dir: str, with_sophus_stub: bool) -> str:
    from beluga_b200 import build as bb_build

    bb_build.build()
    src = os.path.join(ROOT, "tests", "cpp", "test_point_cloud_adaptors.cpp")
    lib_dir = os.path.join(ROOT, "beluga_b200")
    exe = os.path.join(build_dir, "test_point_cloud_adaptors" + ("_sophus" if with_sophus_stub else ""))
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", lib_dir, "-lbeluga_b200", f"-Wl,-rpath,{lib_dir}"]
    if with_sophus_stub:
        cmd[1:1] = ["-DBELUGA_B200_WITH_SOPHUS", "-I", os.path.join(ROOT, "tests", "cpp", "stubs")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return exe


@pytest.mark.parametrize("with_sophus_stub", [False, True])
def test_point_cloud_adaptors_convert_on_the_host(build_dir, with_sophus_stub):
    exe = build_exe(build_dir, with_sophus_stub)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "CPP_POINT_CLOUD_OK" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("with_sophus_stub", [False, True])
def test_point_cloud_adaptors_update_the_filter(build_dir, with_sophus_stub):
    exe = build_exe(build_dir, with_sophus_stub)
    out = subprocess.run([exe, "--gpu"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "CPP_POINT_CLOUD_OK" in out.stdout, out.stdout + out.stderr
