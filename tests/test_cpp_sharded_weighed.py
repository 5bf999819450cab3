"""The C++ adaptor for a caller's device sensor model on shards (include/beluga_b200/amcl.hpp: ShardedAmcl::update with a token that
weighs on the device): compiles with and without the Sophus conversions; run on a machine without a device it reports
BB200_ERR_NO_DEVICE, on the GPU every step of 2 shards equals a twin driven through bb200_sharded_amcl_update_begin / _end
and a standalone Amcl weighed by the same token."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("cpp_sharded_weighed"))


def build_exe(build_dir: str, with_sophus_stub: bool = False) -> str:
    from beluga_b200 import build as bb_build

    bb_build.build()
    lib_dir = os.path.join(ROOT, "beluga_b200")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(shutil.which(bb_build.nvcc()))))  # the toolkit nvcc belongs to
    model = os.path.join(build_dir, "position_fix.o")
    out = subprocess.run([bb_build.nvcc(), "-std=c++17", "-O2", *bb_build.ARCH, "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-c",
                          os.path.join(ROOT, "tests", "cpp", "position_fix.cu"), "-o", model], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    exe = os.path.join(build_dir, "test_sharded_weighed_adaptor" + ("_sophus" if with_sophus_stub else ""))
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "test_sharded_weighed_adaptor.cpp"), model, "-o", exe, "-L", lib_dir, "-lbeluga_b200",
           f"-Wl,-rpath,{lib_dir}", "-L", os.path.join(cuda, "lib64"), "-lcudart", f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}"]
    if with_sophus_stub:
        cmd[1:1] = ["-DBELUGA_B200_WITH_SOPHUS", "-I", os.path.join(ROOT, "tests", "cpp", "stubs")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return exe


def test_sharded_weighed_adaptor_compiles_with_sophus_conversions(build_dir):
    build_exe(build_dir, with_sophus_stub=True)


def test_sharded_weighed_adaptor_without_device(build_dir):
    import beluga_b200 as bb

    if bb.device_count() > 0:
        pytest.skip("a GPU is present")
    out = subprocess.run([build_exe(build_dir)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "SHARDED_WEIGHED_ADAPTOR_NO_DEVICE" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_sharded_weighed_adaptor_runs(build_dir):
    out = subprocess.run([build_exe(build_dir)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "SHARDED_WEIGHED_ADAPTOR_OK" in out.stdout, out.stdout + out.stderr
