"""Ablation of the likelihood-field reweight kernel on the flagship workload (1M particles x 1080 beams, 2000^2 map).

    PYTHONPATH=. python tools/reweight_ablation.py [--variants a,b,c,d] [--runs 3] [--steps 30] [--warmup 5] [--out DIR]
    PYTHONPATH=. python tools/reweight_ablation.py --build-only --out DIR     # compile the variants, no GPU needed

Each variant is the library of this tree with a few source edits, compiled for sm_90a into DIR/<variant>/ (only the edited
sources are recompiled; the rest link from the tree's beluga_b200/build/*.o, so run `python -m beluga_b200.build` first).
The runs alternate the variants round by round, one process per run, and each run times `--steps` fused steps with the L2
flushed (256 MiB device write) before every step, like bench.py.  Per run: the mean of every kernel's CUDA-event time,
the median SM clock, clock-event reasons seen during the run, and the card's name and power limit.

Variants:
  a  the kernel as it is
  b  warm table: the L2 prefetch of the table run again by a launch just before the reweight (own timing mark
     "warm_table"), a bound on what keeping the table in L2 through the step can gain
  c  the persistent kernel with the scan staged once per CTA into shared memory by TMA bulk copy, read with one LDS.128
     per beam, instead of the constant-bank kernel parameter (scans up to 1920 points)
  d  every gather's index ANDed with a run-time zero (all lanes read element 0 of the bordered table: broadcast L1 hits),
     the instruction stream kept, a ceiling for any change on the gather side
A variant whose edit no longer applies to the tree (its anchor text is gone) is reported and skipped.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (source file under csrc, anchor text, replacement)
_C_PROLOGUE = """const double2* __restrict__ points) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* s_pts = reinterpret_cast<double2*>(smem_raw);
  __shared__ __align__(8) uint64_t s_bar;
  if (threadIdx.x == 0) {
    mbarrier_init(&s_bar, 1);
    mbarrier_init_fence();
    mbarrier_expect_tx(&s_bar, n_points * static_cast<uint32_t>(sizeof(double2)));
    bulk_copy_g2s(s_pts, points, n_points * static_cast<uint32_t>(sizeof(double2)), &s_bar);
  }
  __syncthreads();
  mbarrier_wait(&s_bar, 0);
"""
VARIANTS = {
    "a": [],
    "b": [("filter.cu", '      mark("reweight_lfm");\n',
           '      mark("warm_table");\n'
           "      launch_begin_fused_step(scalars_.get(), tile_state_.get(), 0, nullptr, nullptr, 0, nullptr, 0, map_.field.bordered,\n"
           "                              map_.bordered_bytes, stream_);\n"
           '      mark("reweight_lfm");\n')],
    "c": [("reweight_lfm.cu", "const __grid_constant__ ScanParam scan) {\n", _C_PROLOGUE),
          ("reweight_lfm.cu", "scan.p, n_points, acc);", "s_pts, n_points, acc);"),
          ("reweight_lfm.cu", "<<<persistent, kRwThreads, 0, stream>>>(states, weights, n, perm, field, n_points, points_radius, scalars, scan);",
           "<<<persistent, kRwThreads, smem, stream>>>(states, weights, n, perm, field, n_points, points_radius, scalars, points);")],
    "d": [("reweight_lfm.cuh", "const double* table = kInGrid ? field.bordered_biased : field.bordered;", "const double* table = field.bordered;"),
          ("reweight_lfm.cuh", "acc[k] = acc[k] + fixed_lookup<kInGrid>(kInGrid ? field.bordered_biased : field.bordered,",
           "acc[k] = acc[k] + fixed_lookup<kInGrid>(field.bordered,"),
          ("reweight_lfm.cuh", "  return __ldg(table + idx);\n}\n\n/// The reference's operation sequence",
           "  return __ldg(table + (idx & (g.y_max >> 31)));\n}\n\n/// The reference's operation sequence")],
}
HEADER_UNITS = {"reweight_lfm.cuh": ["reweight_lfm.cu", "batch_kernels.cu"]}


def build_variant(name: str, out_dir: str) -> str | None:
    """Compiles variant `name` into out_dir/name/libbeluga_b200.so; None if an edit does not apply."""
    from beluga_b200 import build as bb

    edits = VARIANTS[name]
    vdir = os.path.join(out_dir, name)
    shutil.rmtree(vdir, ignore_errors=True)
    csrc = os.path.join(vdir, "beluga_b200", "csrc")  # sources include ../../include
    shutil.copytree(bb.CSRC, csrc)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(vdir, "include"))
    touched = set()
    for src, old, new in edits:
        path = os.path.join(csrc, src)
        with open(path) as f:
            text = f.read()
        if text.count(old) < 1:
            print(f"variant {name}: edit of {src} does not apply (anchor {old[:60]!r} not found); skipped", file=sys.stderr)
            return None
        with open(path, "w") as f:
            f.write(text.replace(old, new))
        touched.add(src)
    # a header edit recompiles the sources that include it
    units = set()
    for src in touched:
        units.update(HEADER_UNITS.get(src, [src]))
    objs = []
    for s in bb.SOURCES:
        base = os.path.splitext(s)[0] + ".o"
        if s in units:
            obj = os.path.join(vdir, base)
            cmd = [bb.nvcc(), *bb.NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(csrc, s), "-o", obj]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"variant {name}: {s} failed to compile:\n{r.stdout}{r.stderr}")
            with open(os.path.join(vdir, "ptxas.txt"), "a") as f:
                f.write(f"--- {s}\n{r.stdout}{r.stderr}\n")
        else:
            obj = os.path.join(bb.HERE, "build", base)
            if not os.path.exists(obj):
                raise RuntimeError(f"{obj} missing: run `python -m beluga_b200.build` first")
        objs.append(obj)
    lib = os.path.join(vdir, "libbeluga_b200.so")
    subprocess.run([bb.nvcc(), "-shared", *bb.ARCH, "-cudart", "static", "-o", lib, *objs, "-ccbin", "/usr/bin/g++"], check=True)
    return lib


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


class Clocks:
    """SM clock and clock-event reasons, sampled with NVML every 10 ms while the timed steps run."""

    def __init__(self):
        import pynvml

        pynvml.nvmlInit()
        self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(0)
        self.sm, self.reasons = [], set()
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        names = {0x4: "sw_power_cap", 0x8: "hw_slowdown", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown"}
        while not self._stop.is_set():
            self.sm.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
            mask = self.nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
            self.reasons.update(n for bit, n in names.items() if mask & bit)
            self._stop.wait(0.01)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join(timeout=5)


def worker(lib: str, scenario_path: str, steps: int, warmup: int) -> dict:
    import numpy as np
    import torch

    from beluga_b200 import _capi

    _capi.LIB_PATH = lib
    import beluga_b200 as bb

    z = np.load(scenario_path, allow_pickle=False)
    poses, scans = z["poses"], [z[f"scan{k}"] for k in range(len(z["poses"]))]
    amcl = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05),
                   bb.AmclParams(min_particles=1_000_000, max_particles=1_000_000, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1))
    amcl.update_map(bb.SENSOR_LIKELIHOOD_FIELD,
                    bb.LikelihoodFieldModelParam(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2),
                    bb.OccupancyGrid(z["cells"], float(z["resolution"])))
    amcl.initialize(z["initial_mean"], z["initial_cov"])
    filt = amcl.filter
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    filt.set_timing(True)
    k = 0

    def step():
        nonlocal k
        r = amcl.update(bb.se2(*poses[k % len(poses)]), np.ascontiguousarray(scans[k % len(poses)]))
        assert r.updated == 1
        k += 1

    for _ in range(warmup):
        step()
    kernel_ms = {}
    with Clocks() as clocks:
        for _ in range(steps):
            flush.zero_()
            torch.cuda.synchronize()
            filt.clear_timings()
            step()
            per = {}
            for name, ms in filt.last_timings():
                per[name] = per.get(name, 0.0) + ms
            for name, ms in per.items():
                kernel_ms.setdefault(name, []).append(ms)
    torch.cuda.synchronize()
    means = {n: float(np.mean(v)) for n, v in kernel_ms.items()}
    return {"kernels_ms": means, "step_ms": sum(means.values()), "sm_mhz": float(np.median(clocks.sm)) if clocks.sm else None,
            "reasons": sorted(clocks.reasons)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", default="a,b,c,d")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="variant builds (default: a temporary directory)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--worker", nargs=2, metavar=("LIB", "SCENARIO"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        print(json.dumps(worker(args.worker[0], args.worker[1], args.steps, args.warmup)), flush=True)
        return
    out = args.out or tempfile.mkdtemp(prefix="reweight_ablation_")
    os.makedirs(out, exist_ok=True)
    libs = {}
    for v in args.variants.split(","):
        lib = os.path.join(out, v, "libbeluga_b200.so")
        if not os.path.exists(lib):
            lib = build_variant(v, out)
        if lib is not None:
            libs[v] = lib
    if args.build_only:
        print(json.dumps(libs))
        return
    from beluga_b200 import synthetic
    import numpy as np

    sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=100)
    scen = os.path.join(tempfile.mkdtemp(prefix="reweight_ablation_scene_"), "scenario.npz")
    np.savez(scen, cells=sc.cells, resolution=sc.resolution, poses=sc.poses, initial_mean=sc.initial_mean, initial_cov=sc.initial_cov,
             **{f"scan{k}": s for k, s in enumerate(sc.scans)})
    results = {v: [] for v in libs}
    info = card()
    for rnd in range(args.runs):
        for v, lib in libs.items():
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", lib, scen, "--steps", str(args.steps), "--warmup", str(args.warmup)],
                               capture_output=True, text=True, cwd=ROOT)
            if r.returncode != 0:
                print(f"variant {v} run {rnd}: exit {r.returncode}\n{r.stdout[-2000:]}{r.stderr[-4000:]}", file=sys.stderr)
                continue
            res = json.loads(r.stdout.strip().splitlines()[-1])
            results[v].append(res)
            print(json.dumps({"variant": v, "run": rnd, "reweight_lfm_ms": res["kernels_ms"].get("reweight_lfm"), **res}), flush=True)
    summary = {"card": info, "steps": args.steps, "warmup": args.warmup, "variants": {}}
    for v, rs in results.items():
        rw = [r["kernels_ms"]["reweight_lfm"] for r in rs]
        summary["variants"][v] = {"reweight_lfm_ms": rw, "step_ms": [r["step_ms"] for r in rs], "sm_mhz": [r["sm_mhz"] for r in rs],
                                  "reasons": sorted({x for r in rs for x in r["reasons"]}),
                                  "warm_table_ms": [r["kernels_ms"].get("warm_table") for r in rs]}
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
