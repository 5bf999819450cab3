"""The header-only C++ adaptors (include/beluga_b200/*.hpp): compile on CPU, run the reference's
beluga::Amcl smoke tests through them on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    """Executables go to a temporary directory: the checkout may be read-only."""
    return str(tmp_path_factory.mktemp("cpp_adaptors"))


def build_exe(build_dir: str, with_sophus_stub: bool = False) -> str:
    from beluga_b200 import build as bb_build

    bb_build.build()
    src = os.path.join(ROOT, "tests", "cpp", "test_adaptors.cpp")
    lib_dir = os.path.join(ROOT, "beluga_b200")
    exe = os.path.join(build_dir, "test_adaptors" + ("_sophus" if with_sophus_stub else ""))
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", lib_dir, "-lbeluga_b200", f"-Wl,-rpath,{lib_dir}"]
    if with_sophus_stub:  # Sophus/Eigen are absent here: 30-line stand-ins type-check the BELUGA_B200_WITH_SOPHUS conversion path
        cmd[1:1] = ["-DBELUGA_B200_WITH_SOPHUS", "-I", os.path.join(ROOT, "tests", "cpp", "stubs")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return exe


def test_adaptors_compile_with_sophus_conversions(build_dir):
    build_exe(build_dir, with_sophus_stub=True)


def test_adaptors_compile(build_dir):
    assert os.path.exists(build_exe(build_dir))


@pytest.mark.gpu
def test_adaptors_run_reference_smoke_tests(build_dir):
    exe = build_exe(build_dir)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "CPP_ADAPTORS_OK" in out.stdout, out.stdout + out.stderr
