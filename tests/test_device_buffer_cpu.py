"""csrc/device_buffer.hpp on the CPU: the owner of every device and pinned buffer of the library.

The header needs nothing from CUDA but <cuda_runtime_api.h>, so g++ compiles it against a test (tests/cpp/test_device_buffer.cpp)
that defines cudaMalloc, cudaFree, cudaMallocHost, cudaFreeHost and cudaMemcpyAsync itself, over malloc, and links no CUDA
runtime.  The test counts the live allocations, fails the k-th allocation on request and records every copy; it checks that

* the destructor and moves free every buffer exactly once, each with the free of its kind;
* allocate(0) still allocates one element, and grow() reallocates only when the buffer holds fewer elements than asked;
* a failed allocate() or grow() leaves the buffer null with size 0 and nothing live;
* a group of buffers allocated into a local struct and moved into its owner on success is all or nothing: a failure at
  any of its allocations leaves the owner's buffers as they were and frees whatever the attempt allocated;
* a MirroredBuffer grows both halves, reports the smaller half's size after a failed one and grows that half again on
  the next call, frees each half once through moves, and copies exactly the element range asked for, in the direction
  asked for, returning the copy's error.
"""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INCLUDE = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


def test_device_buffer_owns_and_groups_allocate_all_or_nothing():
    out_dir = os.path.join(ROOT, "tests", "cpp", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_device_buffer")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + CUDA_INCLUDE, "-o", exe,
           os.path.join(ROOT, "tests", "cpp", "test_device_buffer.cpp")]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-3000:]
    ran = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert ran.returncode == 0, ran.stdout[-3000:] + ran.stderr[-3000:]
    assert "all device buffer checks passed" in ran.stdout
