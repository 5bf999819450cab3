"""csrc/shard_link.cpp on the CPU: the link between the shards of one filter and the CUDA IPC mappings it owns.

g++ compiles the link against a test (tests/cpp/test_shard_link.cpp) that defines the CUDA functions it calls itself and
links no CUDA runtime.  The stub cudaIpcOpenMemHandle / cudaIpcCloseMemHandle count the live mappings and fail the k-th
open on request; the test checks that

* a join over CUDA IPC of 2, 3 and 8 ranks, with and without the KLD hash arrays, opens each peer's handles once and never
  this rank's own handles or a peer's empty KLD handle, and that the views put this rank's own buffers at its rank;
* a failure at any single open leaves the link unjoined with no live mapping, and the link can join afterwards;
* leave() and destruction close every mapping exactly once, and a second leave() closes nothing;
* a join of shards in one process borrows the other links' buffers and closes nothing.
"""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INCLUDE = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


def test_shard_link_owns_its_ipc_mappings_and_joins_all_or_nothing():
    out_dir = os.path.join(ROOT, "tests", "cpp", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_shard_link")
    # -Wno-unknown-pragmas: se2_math.cuh, reached through kernels.cuh, carries a device-only #pragma unroll
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-Wno-unknown-pragmas", "-I" + CUDA_INCLUDE, "-o", exe,
           os.path.join(ROOT, "tests", "cpp", "test_shard_link.cpp"), os.path.join(ROOT, "beluga_b200", "csrc", "shard_link.cpp")]
    built = subprocess.run(cmd, capture_output=True, text=True)
    assert built.returncode == 0, built.stderr[-3000:]
    ran = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert ran.returncode == 0, ran.stdout[-3000:] + ran.stderr[-3000:]
    assert "all shard link checks passed" in ran.stdout
