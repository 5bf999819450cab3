"""Builds libbeluga_b200.so (CUDA kernels + C ABI) in-tree for sm_90a (H100) with nvcc.

    python -m beluga_b200.build [--force]

-fmad=false / -ffp-contract=off: the reference pipeline is built for baseline x86-64 and rounds
after every multiply; the likelihood-field cell a beam lands in must not depend on contraction.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbeluga_b200.so")
SOURCES = ["step.cu", "propagate.cu", "reweight_lfm.cu", "reweight_beam.cu", "reweight_landmark.cu", "raycast.cu", "cdf.cu", "kld.cu", "resample.cu", "batch_kernels.cu",
           "shard_exchange.cu", "cluster.cu", "cluster_select.cu", "device_map.cu", "filter.cu", "amcl.cu", "sharded_amcl.cu", "batch.cu", "c_api.cu", "shard_link.cpp", "map_host.cpp", "cluster_host.cpp", "state_blob.cpp"]
HEADERS = ["kernels.cuh", "device_common.cuh", "bucket_set.cuh", "kld.cuh", "propagate.cuh", "reweight_lfm.cuh", "reweight_beam.cuh", "reweight_landmark.cuh", "reweight_landmark_block.cuh", "raycast.cuh", "cdf.cuh", "resample.cuh",
           "cluster.cuh", "cluster_select.cuh", "cluster_host.hpp", "se2_math.cuh", "device_buffer.hpp", "device_map.hpp", "shard_link.hpp", "filter.hpp", "amcl.hpp", "sharded_amcl.hpp", "batch.hpp", "map_host.hpp", "measurement_host.hpp", "state_blob.hpp",
           os.path.join("..", "..", "include", "beluga_b200.h")]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    *ARCH,
    "-fmad=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-Wall",
    "-ccbin", "/usr/bin/g++",
]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if src.endswith(".cu") and verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.run([nvcc(), "-shared", *ARCH, "-cudart", "static", "-o", LIB, *objs, "-ccbin", "/usr/bin/g++"], check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
