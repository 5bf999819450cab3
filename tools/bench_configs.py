#!/usr/bin/env python
"""Timings of the other BASELINE.json configurations (parity-test cases, not the bench.py line), and of point-cloud updates:
`cloud`: 65 536-point lidar clouds at 10k and 1M particles.  `batch`: K node-sized filters (2000 particles x 100 points) stepped as one
AmclBatch against K standalone Amcl stepped one after another.  `batch_cluster`: the same batches with the beluga_ros-shaped round
update + cluster estimate, the estimate taken for all members in one call and member by member.  `batch_beam`: AmclBatch with the
beam model (60 and 720 points per member) against the same members stepped as standalone Amcl.  `batch_maps`: one AmclBatch whose
members read 1, 4 or 16 likelihood-field maps against one single-map batch per map, and a step mixing likelihood-field and beam members.
`batch_cloud`: the `batch` members' particle-cloud publish round (histograms and pose samples) in one batched call each against
K standalone filters publishing in turn.  `batch_measurements`: AmclBatch fed laser scans and point clouds converted on the
device against host conversion plus the points update.  `batch_kld`: the `batch` workload with KLD-adaptive members (min 500,
max 2000) against K standalone KLD Amcl.  `batch_selective`: the `batch` workload with selective-resampling members, fixed-size
and KLD-adaptive (min 500, max 2000), against K standalone selective Amcl.  `batch_members`: add_member and remove_member at
K = 16 and 256 members, alone and next to a 32 768-particle member, and a step after churn against the same step on a fresh batch.
`batch_state`: export_members and AmclBatch.from_states (the fleet checkpoint and its restore) with the same members.
`raycast`: device ray casts (Ray2d::cast) for 256 batch members x 1 pose x 1080 bearings and for 1M rays of one filter, against
the CPU oracle's Ray2d on the same rays.
`weighed`: a 1M-particle step at 1080 beams on the 2000^2 map through the built-in likelihood-field update, against the same
step weighed by the caller (bb200_amcl_update_begin, a one-kernel torch weigh on the step's stream, bb200_amcl_update_end);
and a 256 x 2000 batch through update_measurements (100 points per member) against bb200_amcl_batch_update_begin / _end
with every member weighed by one torch kernel.
`sharded-publish`: a 1M-particle filter's publish round (particle-cloud histogram and 2000 pose samples) and 1M ray casts on 2
and 4 shards of one device, next to the single filter (a filter of one shard does not step, so it has no posterior to publish).
`sharded-weighed`: a 1M-particle step at 1080 beams on the 2000^2 map through the built-in likelihood-field update against the
same step weighed by the caller (update_weighted, one torch kernel per shard), on one filter and on 2 and 4 shards of device 0
(and over devices 0..1 and 0..3 where there are that many).
`landmark`: the landmark and bearing models at 1M particles x 16 detections on a fiducial-like and a reflector-like map, with
the reweight kernel's share of the FP64 bound and the Python oracle beside them.
`batch_landmark`: AmclBatch with the landmark model, K in {1, 16, 64, 256} members x 2000 particles x 16 detections on the
same two maps, against the same members stepped as standalone Amcl.update_landmarks.
`sharded_landmark`: `landmark`'s 1M-particle steps on one filter and on 2, 4 and 8 shards of device 0 (what sharding costs),
and over 2, 4 and 8 devices where there are that many (how it scales), with each shard's reweight kernel time.
C1 10k x 180 LFM 500^2 multinomial (GPU and CPU oracle seq/par), C3 1M x 720 beam model 2000^2,
C4 KLD-adaptive 100k..10M LFM.  Writes gpurun_out/configs.json."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import beluga_b200 as bb  # noqa: E402
from beluga_b200 import synthetic  # noqa: E402

MOTION = (0.1, 0.05, 0.1, 0.05)
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)


def run_gpu(sc, sensor, sensor_params, params, steps, warmup=2, clouds=None):
    """`clouds`: one synthetic.PointCloud per step, fed through Amcl.update_point_cloud (conversion included in the step time)."""
    a = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), params)
    a.update_map(sensor, sensor_params, bb.OccupancyGrid(sc.cells, sc.resolution))
    a.initialize(sc.initial_mean, sc.initial_cov)
    a.filter.set_timing(True)
    wall, sizes, kernels = [], [], {}
    for k in range(warmup + steps):
        a.filter.clear_timings()
        pose = bb.se2(*sc.poses[k % 100])
        t0 = time.perf_counter()
        if clouds is None:
            r = a.update(pose, sc.scans[k % 100])
        else:
            pc = clouds[k]
            r = a.update_point_cloud(pose, pc.data, pc.point_step, pc.x_offset, pc.datatype, origin=pc.origin)
        dt = time.perf_counter() - t0
        assert r.updated == 1
        if k >= warmup:
            wall.append(dt * 1e3)
            sizes.append(int(r.n_particles))
            for name, ms in a.filter.last_timings():
                kernels[name] = kernels.get(name, 0.0) + ms / steps
    return {"ms_per_step_e2e": float(np.mean(wall)), "steps_per_s_e2e": 1e3 / float(np.mean(wall)), "particles": sizes,
            "kernels_ms": {k: round(v, 4) for k, v in kernels.items()}}


def device_record():
    """Name and power limit of the card this process measures on (a read-only nvidia-smi query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, check=True)
        name, power, clock = (q.stdout.strip().split(", ") + ["?", "?", "?"])[:3]
    except (OSError, subprocess.CalledProcessError):
        name, power, clock = "nvidia-smi unavailable", "?", "?"
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def run_cloud():
    """Point-cloud updates (Amcl.update_point_cloud) with 64 x 1024 synthetic lidar clouds: 10k particles on C1's 500^2 map (the
    node-sized case) and 1M on C2's 2000^2 map, and beside them C2's 1M x 1080 scan in the same process, so that the reweight
    kernel's lookup rate with 32 shared-memory chunks per particle can be read against the scan's."""
    res = {}
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    cases = (("cloud_10k_x_65536_lfm_500", 500, 10_000, 20, 2), ("cloud_1M_x_65536_lfm_2000", 2000, 1_000_000, 5, 1))
    for name, grid, n, steps, warmup in cases:
        sc = synthetic.make_scenario(grid_size=grid, n_beams=1080, steps=100)
        clouds = [synthetic.make_point_cloud(sc, k, rows=64, azimuths=1024) for k in range(warmup + steps)]
        params = bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1)
        r = run_gpu(sc, bb.SENSOR_LIKELIHOOD_FIELD, lfm, params, steps=steps, warmup=warmup, clouds=clouds)
        r["points"] = 64 * 1024
        r["lookups_per_ns_reweight"] = n * r["points"] / (r["kernels_ms"]["reweight_lfm"] * 1e6)
        res[name] = r
        if grid == 2000:
            scan = run_gpu(sc, bb.SENSOR_LIKELIHOOD_FIELD, lfm, params, steps=10, warmup=3)
            scan["points"] = 1080
            scan["lookups_per_ns_reweight"] = n * 1080 / (scan["kernels_ms"]["reweight_lfm"] * 1e6)
            res["cloud_reference_1M_x_1080_scan_lfm_2000"] = scan
    device = device_record()
    for r in res.values():
        r["device"] = device
    return res


def run_batch():
    """AmclBatch with K in {1, 16, 64, 256} members x 2000 particles x 100 points (the reference benchmark's max_beams) on the 2000^2
    synthetic map, systematic resampling, every member updating every step; beside it, in the same process, K standalone Amcl
    stepped one after another on the same inputs."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    n, steps, warmup = 2000, 20, 3
    device = device_record()
    for k in (1, 16, 64, 256):
        params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
        motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
        batch = bb.AmclBatch(motions, params)
        batch.set_likelihood_field_map(lfm, grid)
        singles = []
        for m in range(k):
            batch.initialize(m, sc.initial_mean, sc.initial_cov)
            a = bb.Amcl(motions[m], params[m])
            a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid)
            a.initialize(sc.initial_mean, sc.initial_cov)
            singles.append(a)
        wall_batch, wall_single, launches = [], [], []
        for t in range(warmup + steps):
            pose = bb.se2(*sc.poses[t])
            t0 = time.perf_counter()
            before = batch.launch_count()
            r = batch.update([pose] * k, [sc.scans[t]] * k)
            t1 = time.perf_counter()
            assert all(x.updated for x in r)
            launches.append(batch.launch_count() - before)
            for a in singles:
                assert a.update(pose, sc.scans[t]).updated == 1
            t2 = time.perf_counter()
            if t >= warmup:
                wall_batch.append((t1 - t0) * 1e3)
                wall_single.append((t2 - t1) * 1e3)
        mb, ms = float(np.median(wall_batch)), float(np.median(wall_single))
        res[f"batch_{k}_x_2000_x_100_lfm_2000"] = {
            "members": k, "particles": n, "points": 100, "steps": steps,
            "ms_per_step_e2e": mb, "member_steps_per_s": k * 1e3 / mb, "launches_per_step": int(max(launches)),
            "standalone_ms_per_round": ms, "standalone_member_steps_per_s": k * 1e3 / ms,
            "kernels_ms": {}, "device": device}
    return res


def run_batch_kld():
    """`batch` with KLD-adaptive members: K in {1, 16, 64, 256} members of min 500 / max 2000 particles (beluga_ros's defaults)
    x 100 points on the 2000^2 synthetic map, every member updating every step; beside it K standalone KLD Amcl stepped one
    after another in the same process."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    steps, warmup = 20, 3
    device = device_record()
    for k in (1, 16, 64, 256):
        params = [bb.AmclParams(min_particles=500, max_particles=2000, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
        motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
        batch = bb.AmclBatch(motions, params, adaptive=True)
        batch.set_likelihood_field_map(lfm, grid)
        singles = []
        for m in range(k):
            batch.initialize(m, sc.initial_mean, sc.initial_cov)
            a = bb.Amcl(motions[m], params[m])
            a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid)
            a.initialize(sc.initial_mean, sc.initial_cov)
            singles.append(a)
        wall_batch, wall_single, launches, sizes = [], [], [], []
        for t in range(warmup + steps):
            pose = bb.se2(*sc.poses[t])
            t0 = time.perf_counter()
            before = batch.launch_count()
            r = batch.update([pose] * k, [sc.scans[t]] * k)
            t1 = time.perf_counter()
            assert all(x.updated for x in r)
            launches.append(batch.launch_count() - before)
            for a, x in zip(singles, r):
                assert a.update(pose, sc.scans[t]).n_particles == x.n_particles
            t2 = time.perf_counter()
            if t >= warmup:
                wall_batch.append((t1 - t0) * 1e3)
                wall_single.append((t2 - t1) * 1e3)
                sizes.extend(x.n_particles for x in r)
        mb, ms = float(np.median(wall_batch)), float(np.median(wall_single))
        res[f"batch_kld_{k}_x_500_2000_x_100_lfm_2000"] = {
            "members": k, "min_particles": 500, "max_particles": 2000, "points": 100, "steps": steps,
            "mean_particles": float(np.mean(sizes)), "ms_per_step_e2e": mb, "member_steps_per_s": k * 1e3 / mb,
            "launches_per_step": int(max(launches)), "standalone_ms_per_round": ms, "standalone_member_steps_per_s": k * 1e3 / ms,
            "kernels_ms": {}, "device": device}
    return res


def run_batch_selective():
    """`batch` with selective-resampling members (on_effective_size_drop): K in {1, 16, 64, 256} members x 2000 particles x 100
    points on the 2000^2 synthetic map, in one arm fixed-size and in the other KLD-adaptive (min 500, max 2000), every member
    updating every step; beside it K standalone selective Amcl stepped one after another in the same process.  Also the share
    of member-steps that resampled."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    steps, warmup = 20, 3
    device = device_record()
    for arm, lo in (("fixed", 2000), ("kld", 500)):
        for k in (1, 16, 64, 256):
            params = [bb.AmclParams(min_particles=lo, max_particles=2000, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m, selective_resampling=True)
                      for m in range(k)]
            motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
            batch = bb.AmclBatch(motions, params, adaptive=lo < 2000, selective=True)
            batch.set_likelihood_field_map(lfm, grid)
            singles = []
            for m in range(k):
                batch.initialize(m, sc.initial_mean, sc.initial_cov)
                a = bb.Amcl(motions[m], params[m])
                a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid)
                a.initialize(sc.initial_mean, sc.initial_cov)
                singles.append(a)
            wall_batch, wall_single, launches, resampled, sizes = [], [], [], [], []
            for t in range(warmup + steps):
                pose = bb.se2(*sc.poses[t])
                t0 = time.perf_counter()
                before = batch.launch_count()
                r = batch.update([pose] * k, [sc.scans[t]] * k)
                t1 = time.perf_counter()
                assert all(x.updated for x in r)
                launches.append(batch.launch_count() - before)
                for a, x in zip(singles, r):
                    y = a.update(pose, sc.scans[t])
                    assert y.resampled == x.resampled and y.n_particles == x.n_particles
                t2 = time.perf_counter()
                if t >= warmup:
                    wall_batch.append((t1 - t0) * 1e3)
                    wall_single.append((t2 - t1) * 1e3)
                    resampled.extend(x.resampled for x in r)
                    sizes.extend(x.n_particles for x in r)
            mb, ms = float(np.median(wall_batch)), float(np.median(wall_single))
            res[f"batch_selective_{arm}_{k}_x_{lo}_2000_x_100_lfm_2000"] = {
                "members": k, "min_particles": lo, "max_particles": 2000, "points": 100, "steps": steps,
                "resampled_share": float(np.mean(resampled)), "mean_particles": float(np.mean(sizes)),
                "ms_per_step_e2e": mb, "member_steps_per_s": k * 1e3 / mb, "launches_per_step": int(max(launches)),
                "standalone_ms_per_round": ms, "standalone_member_steps_per_s": k * 1e3 / ms, "kernels_ms": {}, "device": device}
    return res


def run_batch_members():
    """Members that join and leave: the host-clock time of add_member (a 2000-particle member) and of remove_member, each of
    which ends synchronised, with K in {16, 256} members x 2000 particles holding particles, alone and next to a
    32 768-particle member; and a step of a batch after churn (slot 0 vacated, one member appended) against the same step on
    a freshly created batch of the same members, the two alternated in one session."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    repeats, steps, warmup = 20, 20, 3
    device = device_record()

    def member(m, n=2000):
        return bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m)

    def make(params):
        b = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in params], params)
        b.set_likelihood_field_map(lfm, grid)
        for m in range(len(params)):
            b.initialize(m, sc.initial_mean, sc.initial_cov)
        return b

    for k in (16, 256):
        for big in (False, True):
            params = [member(m) for m in range(k)] + ([member(k, 32768)] if big else [])
            batch = make(params)
            batch.update([bb.se2(*sc.poses[0])] * len(params), [sc.scans[0]] * len(params))
            add_ms, remove_ms, launches = [], [], []
            for r in range(repeats + 1):
                before = batch.launch_count()
                t0 = time.perf_counter()
                slot = batch.add_member(bb.DifferentialDriveModelParam(*MOTION), member(1000 + r))
                t1 = time.perf_counter()
                batch.remove_member(slot)
                t2 = time.perf_counter()
                launches.append(batch.launch_count() - before)
                if r > 0:
                    add_ms.append((t1 - t0) * 1e3)
                    remove_ms.append((t2 - t1) * 1e3)
            live = sum(q.max_particles for q in params)
            res[f"batch_members_change_{k}_x_2000" + ("_and_32768" if big else "")] = {
                "members": len(params), "live_particles": live, "moved_bytes_per_change": 40 * live,  # states and weights: the step resampled, so no CDF is current, and none records ancestors
               
                "add_member_ms": float(np.median(add_ms)), "remove_member_ms": float(np.median(remove_ms)),
                "launches_per_add_and_remove": int(max(launches)), "repeats": repeats,
                "ms_per_step_e2e": float(np.median(add_ms)), "kernels_ms": {}, "device": device}
        churned = make([member(m) for m in range(k)])
        map_id = churned.member_map(0)
        slot = churned.add_member(bb.DifferentialDriveModelParam(*MOTION), member(k))
        churned.remove_member(0)
        churned.update_map(slot, map_id)
        churned.initialize(slot, sc.initial_mean, sc.initial_cov)
        fresh = make([member(m) for m in range(1, k + 1)])
        wall_churned, wall_fresh = [], []
        for t in range(warmup + steps):
            pose = bb.se2(*sc.poses[t])
            t0 = time.perf_counter()
            a = churned.update([pose] * (k + 1), [None] + [sc.scans[t]] * k)
            t1 = time.perf_counter()
            b = fresh.update([pose] * k, [sc.scans[t]] * k)
            t2 = time.perf_counter()
            assert all(x.updated for x in a[1:]) and all(x.updated for x in b)
            if t >= warmup:
                wall_churned.append((t1 - t0) * 1e3)
                wall_fresh.append((t2 - t1) * 1e3)
        mc, mf = float(np.median(wall_churned)), float(np.median(wall_fresh))
        res[f"batch_members_step_after_churn_{k}_x_2000_x_100_lfm_2000"] = {
            "members": k, "steps": steps, "ms_per_step_e2e": mc, "fresh_batch_ms_per_step": mf, "churned_over_fresh": mc / mf,
            "kernels_ms": {}, "device": device}
    return res


def run_batch_state():
    """State blobs: the host-clock time of export_members (every member's blob, one launch, one copy and one
    synchronisation) and of AmclBatch.from_states (a new batch from those blobs: its allocations, one copy and one launch),
    with K in {16, 256} members x 2000 particles that have stepped once, alone and next to a 32 768-particle member; through
    the Python wrappers (bytes in and out) and through the C ABI into buffers allocated once."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=10)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    repeats = 20
    device = device_record()

    def member(m, n=2000):
        return bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m)

    for k in (16, 256):
        for big in (False, True):
            params = [member(m) for m in range(k)] + ([member(k, 32768)] if big else [])
            batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in params], params)
            batch.set_likelihood_field_map(lfm, grid)
            for m in range(len(params)):
                batch.initialize(m, sc.initial_mean, sc.initial_cov)
            batch.update([bb.se2(*sc.poses[0])] * len(params), [sc.scans[0]] * len(params))
            export_ms, create_ms, launches = [], [], []
            for r in range(repeats + 1):
                before = batch.launch_count()
                t0 = time.perf_counter()
                blobs = batch.export_members()
                t1 = time.perf_counter()
                restored = bb.AmclBatch.from_states(blobs)
                t2 = time.perf_counter()
                launches.append((batch.launch_count() - before, restored.launch_count()))
                restored.close()
                if r > 0:
                    export_ms.append((t1 - t0) * 1e3)
                    create_ms.append((t2 - t1) * 1e3)
            # The same two calls through the C ABI into buffers allocated once: the library's share of the times above.
            lib, kk = batch._lib, len(params)
            sizes = (ctypes.c_uint64 * kk)(*[len(b) for b in blobs])
            bufs = [ctypes.create_string_buffer(len(b)) for b in blobs]
            out = (ctypes.c_void_p * kk)(*[ctypes.cast(b, ctypes.c_void_p) for b in bufs])
            data = (ctypes.c_void_p * kk)(*[ctypes.cast(b, ctypes.c_void_p) for b in bufs])
            c_export_ms, c_create_ms = [], []
            for r in range(repeats + 1):
                h = ctypes.c_void_p()
                t0 = time.perf_counter()
                assert lib.bb200_amcl_batch_export_members(batch._h, None, out, sizes, sizes) == 0
                t1 = time.perf_counter()
                assert lib.bb200_amcl_batch_create_from_states(data, sizes, kk, 0, 0, ctypes.byref(h)) == 0
                t2 = time.perf_counter()
                lib.bb200_amcl_batch_destroy(h)
                if r > 0:
                    c_export_ms.append((t1 - t0) * 1e3)
                    c_create_ms.append((t2 - t1) * 1e3)
            live = sum(q.max_particles for q in params)
            res[f"batch_state_{k}_x_2000" + ("_and_32768" if big else "")] = {
                "members": len(params), "live_particles": live, "blob_bytes": sum(len(b) for b in blobs),
                "moved_bytes": 40 * live,  # states and weights: the step resampled, so no CDF is current, and none records ancestors
                "export_members_ms": float(np.median(export_ms)), "create_from_states_ms": float(np.median(create_ms)),
                "export_members_c_ms": float(np.median(c_export_ms)), "create_from_states_c_ms": float(np.median(c_create_ms)),
                "launches_export_and_create": [int(x) for x in max(launches)], "repeats": repeats,
                "ms_per_step_e2e": float(np.median(export_ms)), "kernels_ms": {}, "device": device}
    return res


def run_raycast():
    """Ray casts on the 2000^2 synthetic map (likelihood-field map, 5 cm cells) at 30 m and 60 m: the expected scans of 256
    batch members, one pose x 1080 bearings each (a fleet's health check, or a simulator's tick), in one
    AmclBatch.cast_rays call; and 1M rays (1000 poses x 1000 bearings) through one bb200_filter_cast_rays.  Host clock around
    each call (it ends synchronised; inputs and outputs cross PCIe inside it), median of `repeats` after one warm-up call that
    also builds and uploads the map's free-distance table.  Beside them the CPU oracle's Ray2d::cast on the same rays, one
    thread (tests/_raycast_oracle.py, -O3)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _raycast_oracle  # noqa: E402

    _raycast_oracle.lib()  # compiled before anything is timed

    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    rng = np.random.default_rng(5)
    device = device_record()
    repeats = 20
    bearings = bb.scan_bearings(-np.pi, 2 * np.pi / 1080, 1080)
    k = 256
    params = [bb.AmclParams(min_particles=500, max_particles=500, seed=m) for m in range(k)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)], params)
    batch.set_likelihood_field_map(lfm, grid)
    member_poses = [bb.se2(*sc.poses[rng.integers(0, 100)])[None] for _ in range(k)]
    f = bb.Filter(capacity=16)
    f.set_likelihood_field_map(lfm, grid)
    poses_1m = np.stack([bb.se2(*sc.poses[i % 100]) for i in range(1000)])
    bearings_1m = np.stack([[np.cos(t), np.sin(t)] for t in np.linspace(-np.pi, np.pi, 1000, endpoint=False)])
    # The batch call through the C ABI into arrays built once: the library's share of the Python wrapper's time.
    d = ctypes.POINTER(ctypes.c_double)
    flat = np.ascontiguousarray(np.concatenate(member_poses))
    ranges_c = np.zeros((k, 1080))
    c_args = ((d * k)(*[flat[m:].ctypes.data_as(d) for m in range(k)]), (ctypes.c_uint64 * k)(*[1] * k),
              (d * k)(*[bearings.ctypes.data_as(d)] * k), (ctypes.c_uint64 * k)(*[1080] * k),
              (d * k)(*[ranges_c[m].ctypes.data_as(d) for m in range(k)]))

    def batch_c(max_range):
        p, n_p, b, n_b, r = c_args
        assert batch._lib.bb200_amcl_batch_cast_rays(batch._h, None, None, p, n_p, b, n_b, (ctypes.c_double * k)(*[max_range] * k), r) == 0

    for max_range in (30.0, 60.0):
        batch_c(max_range)
        c_ms = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            batch_c(max_range)
            c_ms.append((time.perf_counter() - t0) * 1e3)
        cases = (("batch_256_x_1_x_1080", lambda: batch.cast_rays(member_poses, bearings, max_range), batch.launch_count, k * 1080,
                  np.concatenate(member_poses), bearings),
                 ("filter_1000_x_1000", lambda: f.cast_rays(poses_1m, bearings_1m, max_range), f.launch_count, 1000 * 1000, poses_1m, bearings_1m))
        for name, call, launches, rays, p, b in cases:
            out = call()  # warm-up (the first call on this map builds its free-distance table)
            times, counts = [], []
            for _ in range(repeats):
                before = launches()
                t0 = time.perf_counter()
                call()
                times.append((time.perf_counter() - t0) * 1e3)
                counts.append(launches() - before)
            t0 = time.perf_counter()
            want = _raycast_oracle.cast_rays(grid.cells, grid.resolution, grid.origin, p, b, max_range)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            got = np.concatenate(out) if isinstance(out, list) else out
            ms = float(np.median(times))
            res[f"raycast_{name}_{int(max_range)}m_2000"] = {
                "rays": rays, "ms_per_call": ms, "ms_per_call_min_max": [float(min(times)), float(max(times))],
                "rays_per_s": rays / (ms * 1e-3), "launches_per_call": int(max(counts)), "repeats": repeats,
                "hit_fraction": float(np.isfinite(got).mean()), "equal_to_oracle": bool(np.array_equal(got.reshape(want.shape), want)),
                "cpu_oracle_ms_one_thread": cpu_ms, "cpu_oracle_rays_per_s": rays / (cpu_ms * 1e-3),
                "ms_per_step_e2e": ms, "kernels_ms": {}, "device": device}
        res[f"raycast_batch_256_x_1_x_1080_{int(max_range)}m_2000"]["ms_per_call_c"] = float(np.median(c_ms))
    return res


def run_weighed():
    """The built-in likelihood-field update against a weighed step (update_begin, torch.exp(x) into the factors on the step's
    stream, update_end), 1M particles x 1080 beams on the 2000^2 map, systematic resampling every step: the fused path with
    one synchronisation on both sides.  Two filters stepped alternately in one process, host clock around each call (both
    end synchronised), median and range of `steps` after `warmup`.  Then a pass with the device timers on for the kernel
    times; apply_factors moves 24 bytes per particle (w and the factor read, w written)."""
    import torch

    sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=100)
    n = 1_000_000
    params = bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1)
    builtin, weighed = (bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), params) for _ in range(2))
    for a in (builtin, weighed):
        a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(sc.cells, sc.resolution))
        a.initialize(sc.initial_mean, sc.initial_cov)

    def weigh(states, factors):
        torch.exp(states[:, 2], out=factors)

    warmup, steps = 3, 30
    times = {"builtin": [], "weighed": []}
    for k in range(warmup + steps):
        pose = bb.se2(*sc.poses[k % 100])
        for name, call in (("builtin", lambda: builtin.update(pose, sc.scans[k % 100])), ("weighed", lambda: weighed.update_weighted(pose, weigh))):
            t0 = time.perf_counter()
            r = call()
            dt = (time.perf_counter() - t0) * 1e3
            assert r.updated == 1 and r.resampled == 1
            if k >= warmup:
                times[name].append(dt)
    kernels = {"builtin": {}, "weighed": {}}
    timed = 5
    for a in (builtin, weighed):
        a.filter.set_timing(True)
    for k in range(timed):
        pose = bb.se2(*sc.poses[(warmup + steps + k) % 100])
        for name, a, call in (("builtin", builtin, lambda: builtin.update(pose, sc.scans[(warmup + steps + k) % 100])),
                              ("weighed", weighed, lambda: weighed.update_weighted(pose, weigh))):
            a.filter.clear_timings()
            call()
            for kname, ms in a.filter.last_timings():
                kernels[name][kname] = kernels[name].get(kname, 0.0) + ms / timed
    apply_ms = kernels["weighed"].get("apply_factors", float("nan"))
    device = device_record()
    res = {}
    for name in ("builtin", "weighed"):
        t = times[name]
        res[f"weighed_1M_x_1080_lfm_2000_{name}"] = {
            "ms_per_step_e2e": float(np.median(t)), "ms_per_step_min_max": [float(min(t)), float(max(t))], "steps": steps, "warmup": warmup,
            "kernels_ms": {k: round(v, 4) for k, v in kernels[name].items()}, "device": device}
    res["weighed_1M_x_1080_lfm_2000_weighed"].update({"apply_factors_bytes": 24 * n, "apply_factors_gbs": 24 * n / (apply_ms * 1e-3) / 1e9})

    # A 256 x 2000 batch: update_measurements with 100 points per member against begin / end with every member weighed
    # by one torch kernel per member, alternated in one session.
    k, m_n = 256, 2000
    bparams = [bb.AmclParams(min_particles=m_n, max_particles=m_n, seed=m, resample_scheme=bb.RESAMPLE_SYSTEMATIC) for m in range(k)]
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    batches = {}
    for name in ("builtin", "weighed"):
        b = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)], bparams)
        b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(k):
            b.initialize(m, sc.initial_mean, sc.initial_cov)
        batches[name] = b
    pts = [sc.scans[i % 100][::10] for i in range(100)]

    def weigh_batch(members, states, factors):
        for s, f in zip(states, factors):
            torch.exp(s[:, 2], out=f)

    btimes = {"builtin": [], "weighed": []}
    blaunch = {}
    for step in range(warmup + steps):
        poses = np.stack([bb.se2(*sc.poses[step % 100])] * k)
        calls = (("builtin", lambda: batches["builtin"].update_measurements(poses, [pts[step % 100]] * k)),
                 ("weighed", lambda: batches["weighed"].update_weighted(poses, [None] * k, weigh_batch)))
        for name, call in calls:
            before = batches[name].launch_count()
            t0 = time.perf_counter()
            r = call()
            dt = (time.perf_counter() - t0) * 1e3
            assert all(x.updated == 1 for x in r)
            blaunch[name] = batches[name].launch_count() - before
            if step >= warmup:
                btimes[name].append(dt)
    for name in ("builtin", "weighed"):
        t = btimes[name]
        res[f"weighed_batch_256_x_2000_{name}"] = {
            "ms_per_step_e2e": float(np.median(t)), "ms_per_step_min_max": [float(min(t)), float(max(t))], "steps": steps, "warmup": warmup,
            "library_launches_per_step": blaunch[name], "kernels_ms": {}, "device": device}
    return res


def run_sharded_weighed():
    """The built-in sharded step against the weighed sharded step (update_weighted with torch.exp(x) into each shard's factors
    on its stream), 1M particles x 1080 beams on the 2000^2 map, systematic resampling every step.  One shard does not step
    (a filter of one shard has no peers to exchange with): the one-shard row is the standalone Amcl.  Then 2 and 4 shards of
    device 0, and 2 and 4 devices when there are that many.  The built-in and the weighed filter are stepped alternately in
    one process, host clock around each call (both end synchronised), median and range of `steps` after `warmup`; the
    per-shard launch counts of the last step."""
    import torch

    sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=100)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    n, warmup, steps = 1_000_000, 3, 30
    params = bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1)

    def weigh(states, factors):
        torch.exp(states[:, 2], out=factors)

    layouts = [("1_shard", None), ("2_shards", [0, 0]), ("4_shards", [0, 0, 0, 0])]
    layouts += [(f"{k}_devices", list(range(k))) for k in (2, 4) if bb.device_count() >= k]
    device = device_record()
    res = {}
    for name, devices in layouts:
        filters = {}
        for kind in ("builtin", "weighed"):
            f = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), params) if devices is None else bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), params, devices)
            f.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
            f.initialize(sc.initial_mean, sc.initial_cov)
            filters[kind] = f
        shards = {k: [f.filter] if devices is None else f.shards for k, f in filters.items()}
        times = {"builtin": [], "weighed": []}
        launches = {}
        for k in range(warmup + steps):
            pose = bb.se2(*sc.poses[k % 100])
            calls = (("builtin", lambda: filters["builtin"].update(pose, sc.scans[k % 100])), ("weighed", lambda: filters["weighed"].update_weighted(pose, weigh)))
            for kind, call in calls:
                before = [s.launch_count() for s in shards[kind]]
                t0 = time.perf_counter()
                r = call()
                dt = (time.perf_counter() - t0) * 1e3
                assert r.updated == 1 and r.resampled == 1
                launches[kind] = [s.launch_count() - b for s, b in zip(shards[kind], before)]
                if k >= warmup:
                    times[kind].append(dt)
        for kind in ("builtin", "weighed"):
            t = times[kind]
            res[f"sharded_weighed_1M_x_1080_lfm_2000_{name}_{kind}"] = {
                "shards": 1 if devices is None else len(devices), "devices": [0] if devices is None else devices,
                "ms_per_step_e2e": float(np.median(t)), "ms_per_step_min_max": [float(min(t)), float(max(t))], "steps": steps, "warmup": warmup,
                "launches_per_shard": launches[kind], "kernels_ms": {}, "device": device}
        for f in filters.values():
            f.close()
    return res


def run_sharded_publish():
    """What a node publishes around each update, on 1M particles of the 2000^2 map after one resampling step: the particle-cloud
    histogram (1 mm / 1 mrad buckets, the marker array's) plus 2000 pose samples (the pose array's; the CDF is rebuilt inside
    the call, as it is after every resample), and 1M rays (1000 poses x 1000 bearings, 30 m).  A single Amcl, then one
    ShardedAmcl of 2 and 4 shards on device 0 (one shard refuses to step).  Host clock around each call (every call ends synchronised), median of
    `repeats` after one warm-up call."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=100)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    device = device_record()
    n, repeats = 1_000_000, 20
    params = bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1)
    poses = np.stack([bb.se2(*sc.poses[i % 100]) for i in range(1000)])
    bearings = np.stack([[np.cos(t), np.sin(t)] for t in np.linspace(-np.pi, np.pi, 1000, endpoint=False)])
    reference = {}
    for shards in (0, 2, 4):
        if shards == 0:
            f = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), params)
            histogram, sample = f.filter.particle_histogram, f.filter.sample_states
        else:
            f = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), params, devices=[0] * shards)
            histogram, sample = f.particle_histogram, f.sample_states
        f.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        f.initialize(sc.initial_mean, sc.initial_cov)
        assert f.update(bb.se2(*sc.poses[0]), sc.scans[0]).resampled == 1

        def publish():
            return histogram(1e-3, 1e-3), sample(2000, 0xFFFFFFFF)

        cases = (("publish", publish), ("rays_1000_x_1000_30m", lambda: f.cast_rays(poses, bearings, 30.0)))
        name = "single" if shards == 0 else f"{shards}_shards"
        for case, call in cases:
            out = call()
            times = []
            for _ in range(repeats):
                t0 = time.perf_counter()
                call()
                times.append((time.perf_counter() - t0) * 1e3)
            if shards == 0:
                reference[case] = out
            same = (all(np.array_equal(a, b) for a, b in zip(out[0][:4], reference[case][0][:4])) and np.array_equal(out[1], reference[case][1])
                    if case == "publish" else np.array_equal(out, reference[case]))
            ms = float(np.median(times))
            res[f"sharded_publish_{case}_1M_{name}"] = {
                "ms_per_call": ms, "ms_per_call_min_max": [float(min(times)), float(max(times))], "repeats": repeats,
                "equal_to_single_filter": bool(same), "ms_per_step_e2e": ms, "kernels_ms": {}, "device": device}
        f.close()
    return res


def run_batch_beam():
    """AmclBatch with the beam model (beam_max_range 60 m as in C3): K in {1, 16, 64, 256} members x 2000 particles x 60 points
    (beluga_amcl's default max_beams) and 256 x 2000 x 720 points on the 2000^2 synthetic map, systematic resampling, every
    member updating every step; beside it, in the same process, K standalone Amcl stepped one after another on the same inputs.
    On a build without AmclBatch.set_beam_map only the standalone filters are timed."""
    res = {}
    beam = bb.BeamModelParam(beam_max_range=60.0)
    n, steps, warmup = 2000, 20, 3
    batched = hasattr(bb.AmclBatch, "set_beam_map")
    device = device_record()
    for points, ks in ((60, (1, 16, 64, 256)), (720, (256,))):
        sc = synthetic.make_scenario(grid_size=2000, n_beams=points, steps=warmup + steps)
        grid = bb.OccupancyGrid(sc.cells, sc.resolution)
        for k in ks:
            params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
            motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
            batch = bb.AmclBatch(motions, params) if batched else None
            if batched:
                batch.set_beam_map(beam, grid)
            singles = []
            for m in range(k):
                if batched:
                    batch.initialize(m, sc.initial_mean, sc.initial_cov)
                a = bb.Amcl(motions[m], params[m])
                a.update_map(bb.SENSOR_BEAM, beam, grid)
                a.initialize(sc.initial_mean, sc.initial_cov)
                singles.append(a)
            wall_batch, wall_single, launches = [], [], []
            for t in range(warmup + steps):
                pose = bb.se2(*sc.poses[t])
                t0 = time.perf_counter()
                if batched:
                    before = batch.launch_count()
                    r = batch.update([pose] * k, [sc.scans[t]] * k)
                    assert all(x.updated for x in r)
                    launches.append(batch.launch_count() - before)
                t1 = time.perf_counter()
                for a in singles:
                    assert a.update(pose, sc.scans[t]).updated == 1
                t2 = time.perf_counter()
                if t >= warmup:
                    wall_batch.append((t1 - t0) * 1e3)
                    wall_single.append((t2 - t1) * 1e3)
            ms = float(np.median(wall_single))
            row = {"members": k, "particles": n, "points": points, "beam_max_range": 60.0, "steps": steps,
                   "standalone_ms_per_round": ms, "standalone_member_steps_per_s": k * 1e3 / ms, "ms_per_step_e2e": ms, "kernels_ms": {},
                   "device": device}
            if batched:
                mb = float(np.median(wall_batch))
                row.update({"ms_per_step_e2e": mb, "member_steps_per_s": k * 1e3 / mb, "launches_per_step": int(max(launches))})
            res[f"batch_beam_{k}_x_{n}_x_{points}_beam_2000"] = row
    return res


LANDMARK_SENSOR_POSE = (0.0, 0.0, 1.0, 0.2, -1.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.5)


def landmark_maps():
    """The two maps of `landmark` and `sharded_landmark`, each with its 16 detections: (name, positions, categories,
    detection positions, detection categories)."""
    rng = np.random.default_rng(9)
    nd = 16
    for map_name, n_lm, n_cat in (("64_in_64_categories", 64, 64), ("1000_in_1_category", 1000, 1)):
        pos = np.stack([rng.uniform(-20, 20, n_lm), rng.uniform(-20, 20, n_lm), rng.uniform(0, 2, n_lm)], axis=1)
        cat = (np.arange(n_lm) % n_cat).astype(np.uint32)
        det_pos = np.stack([rng.uniform(-5, 5, nd), rng.uniform(-5, 5, nd), rng.uniform(0, 2, nd)], axis=1)
        det_cat = rng.integers(0, n_cat, nd).astype(np.uint32)
        yield map_name, pos, cat, det_pos, det_cat


def landmark_params(n):
    return bb.AmclParams(update_min_d=0.0, update_min_a=0.0, min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1)


def landmark_setup(f, model, pos, cat):
    """The map of `model` on an Amcl or ShardedAmcl, and the particles of a wide Gaussian."""
    lmap = bb.LandmarkMap(pos, cat)
    if model == "landmark":
        f.update_map(bb.SENSOR_LANDMARK, bb.LandmarkModelParam(0.5, 0.3, 1e-3), lmap)
    else:
        f.update_map(bb.SENSOR_BEARING, bb.BearingModelParam(0.3, LANDMARK_SENSOR_POSE), lmap)
    f.initialize([0.0, 0.0, 0.0], np.diag([25.0, 25.0, 1.0]))


def run_landmark():
    """The landmark and bearing models at 1M particles x 16 detections, on (a) 64 landmarks in 64 categories (fiducial-like:
    one candidate per detection) and (b) 1000 landmarks in one category (reflector-like: every detection scans all 1000).
    Amcl.update_landmarks with systematic resampling every step: the host clock around each step (it ends synchronised),
    median of `steps` after `warmup`, with the device timers on for the reweight kernel's time.  The kernel's operation count
    is computed from the shapes: per candidate, the FP64 add, subtract and multiply instructions of the search key (8 for the
    landmark model; 28 for the bearing model, plus its sqrt and three divisions, which are counted once each), over the H100
    SXM's 34 TFLOP/s FP64 rate (an FMA counts two flops there, and the library does not contract, so 17e12 instructions/s).
    Beside it the Python oracle (tests/_landmark_oracle.py, one thread) on 20 particles, scaled to 1M (extrapolated)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _landmark_oracle as lo  # noqa: E402

    res = {}
    device = device_record()
    n, steps, warmup = 1 << 20, 10, 2
    for map_name, pos, cat, det_pos, det_cat in landmark_maps():
        candidates = sum(int((cat == c).sum()) for c in det_cat)
        for model in ("landmark", "bearing"):
            a = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), landmark_params(n))
            landmark_setup(a, model, pos, cat)
            a.filter.set_timing(True)
            wall, kernels = [], {}
            for k in range(warmup + steps):
                a.filter.clear_timings()
                t0 = time.perf_counter()
                r = a.update_landmarks([np.cos(0.01 * k), np.sin(0.01 * k), 0.05 * k, 0.0], det_pos, det_cat)
                dt = time.perf_counter() - t0
                assert r.updated == 1
                if k >= warmup:
                    wall.append(dt * 1e3)
                    for name, ms in a.filter.last_timings():
                        kernels[name] = kernels.get(name, 0.0) + ms / steps
            kernel_ms = kernels.get("reweight_landmark", float("nan"))
            ops = n * candidates * (8 if model == "landmark" else 32)
            states = a.particles()[0][:20]
            dets = [(*p, int(c)) for p, c in zip(det_pos.tolist(), det_cat.tolist())]
            omap = lo.LandmarkMap([(*p, int(c)) for p, c in zip(pos.tolist(), cat.tolist())])
            t0 = time.perf_counter()
            for s in states.tolist():
                if model == "landmark":
                    lo.landmark_weight(s, dets, omap, 0.5, 0.3, 1e-3)
                else:
                    lo.bearing_weight(s, dets, omap, 0.3, LANDMARK_SENSOR_POSE)
            cpu_ms = (time.perf_counter() - t0) * 1e3 * n / len(states)
            res[f"landmark_{model}_1M_x_16_{map_name}"] = {
                "ms_per_step_e2e": float(np.median(wall)), "ms_per_step_min_max": [float(min(wall)), float(max(wall))],
                "reweight_kernel_ms": kernel_ms, "candidates_per_particle": candidates, "fp64_instructions": ops,
                "fp64_bound_ms": ops / 17e12 * 1e3, "share_of_fp64_bound": ops / 17e12 * 1e3 / kernel_ms,
                "cpu_oracle_ms_one_thread_extrapolated": cpu_ms, "kernels_ms": {k: round(v, 4) for k, v in kernels.items()}, "device": device}
            a.close()
    return res


def run_sharded_landmark():
    """`landmark`'s workload (the same two maps, 16 detections, 1M particles, systematic resampling every step) on one Amcl
    and on one ShardedAmcl of 2, 4 and 8 shards of device 0, and of 2, 4 and 8 devices where there are that many.  Shards
    of one device share its SMs: those rows measure what sharding costs, not how it scales.  Host clock around each
    update_landmarks (it ends synchronised), median of `steps` after `warmup`; each shard's reweight_landmark time from
    its device timers (averaged over the steps), and whether the last particle set equals the single filter's."""
    res = {}
    device = device_record()
    n, steps, warmup = 1 << 20, 10, 2
    layouts = [("single", None)] + [(f"{k}_shards_device_0", [0] * k) for k in (2, 4, 8)]
    layouts += [(f"{k}_devices", list(range(k))) for k in (2, 4, 8) if bb.device_count() >= k]
    for map_name, pos, cat, det_pos, det_cat in landmark_maps():
        for model in ("landmark", "bearing"):
            reference = None
            for name, devices in layouts:
                if devices is None:
                    f = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), landmark_params(n))
                    shards = [f.filter]
                else:
                    f = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), landmark_params(n), devices)
                    shards = f.shards
                landmark_setup(f, model, pos, cat)
                for s in shards:
                    s.set_timing(True)
                wall, reweight = [], [0.0] * len(shards)
                for k in range(warmup + steps):
                    for s in shards:
                        s.clear_timings()
                    t0 = time.perf_counter()
                    r = f.update_landmarks([np.cos(0.01 * k), np.sin(0.01 * k), 0.05 * k, 0.0], det_pos, det_cat)
                    dt = time.perf_counter() - t0
                    assert r.updated == 1 and r.resampled == 1
                    if k >= warmup:
                        wall.append(dt * 1e3)
                        for i, s in enumerate(shards):
                            reweight[i] += dict(s.last_timings()).get("reweight_landmark", float("nan")) / steps
                states, weights = f.particles()
                if reference is None:
                    reference = (states, weights)
                res[f"sharded_landmark_{model}_1M_x_16_{map_name}_{name}"] = {
                    "shards": 1 if devices is None else len(devices), "devices": [0] if devices is None else devices,
                    "scaling": "one filter" if devices is None else ("measured" if len(set(devices)) > 1 else "not measured: the shards share one device"),
                    "ms_per_step_e2e": float(np.median(wall)), "ms_per_step_min_max": [float(min(wall)), float(max(wall))], "steps": steps,
                    "warmup": warmup, "reweight_landmark_ms_per_shard": [round(x, 4) for x in reweight],
                    "equal_to_single_filter": bool(states.tobytes() == reference[0].tobytes() and weights.tobytes() == reference[1].tobytes()),
                    "kernels_ms": {}, "device": device}
                f.close()
    return res


def run_batch_landmark():
    """AmclBatch with the landmark model: K in {1, 16, 64, 256} members x 2000 particles x 16 detections on (a) 64 landmarks
    in 64 categories (fiducial-like) and (b) 1000 landmarks in one category (reflector-like), systematic resampling, every
    member updating every step with its own detections; beside it, in the same process and alternated step by step, the
    same K members stepped as standalone Amcl.update_landmarks one after another.  Host clock around each round (both end
    synchronised), median of `steps` after `warmup`."""
    res = {}
    device = device_record()
    rng = np.random.default_rng(13)
    n, nd, steps, warmup = 2000, 16, 20, 3
    param = bb.LandmarkModelParam(0.5, 0.3, 1e-3)
    for map_name, n_lm, n_cat in (("64_in_64_categories", 64, 64), ("1000_in_1_category", 1000, 1)):
        pos = np.stack([rng.uniform(-20, 20, n_lm), rng.uniform(-20, 20, n_lm), rng.uniform(0, 2, n_lm)], axis=1)
        cat = (np.arange(n_lm) % n_cat).astype(np.uint32)
        lmap = bb.LandmarkMap(pos, cat)
        for k in (1, 16, 64, 256):
            params = [bb.AmclParams(update_min_d=0.0, update_min_a=0.0, min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC,
                                    seed=m) for m in range(k)]
            motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
            batch = bb.AmclBatch(motions, params)
            batch.set_landmark_map(param, lmap)
            singles = []
            for m in range(k):
                batch.initialize(m, [0.0, 0.0, 0.0], np.diag([4.0, 4.0, 0.5]))
                a = bb.Amcl(motions[m], params[m])
                a.update_map(bb.SENSOR_LANDMARK, param, lmap)
                a.initialize([0.0, 0.0, 0.0], np.diag([4.0, 4.0, 0.5]))
                singles.append(a)
            wall_batch, wall_single, launches = [], [], []
            for t in range(warmup + steps):
                pose = [np.cos(0.01 * t), np.sin(0.01 * t), 0.05 * t, 0.0]
                dets = [(np.stack([rng.uniform(-5, 5, nd), rng.uniform(-5, 5, nd), rng.uniform(0, 2, nd)], axis=1),
                         rng.integers(0, n_cat, nd).astype(np.uint32)) for _ in range(k)]
                meas = [bb.Detections(*d) for d in dets]
                t0 = time.perf_counter()
                before = batch.launch_count()
                r = batch.update_measurements([pose] * k, meas)
                assert all(x.updated for x in r)
                launches.append(batch.launch_count() - before)
                t1 = time.perf_counter()
                for a, d in zip(singles, dets):
                    assert a.update_landmarks(pose, *d).updated == 1
                t2 = time.perf_counter()
                if t >= warmup:
                    wall_batch.append((t1 - t0) * 1e3)
                    wall_single.append((t2 - t1) * 1e3)
            mb, ms = float(np.median(wall_batch)), float(np.median(wall_single))
            res[f"batch_landmark_{k}_x_{n}_x_{nd}_{map_name}"] = {
                "members": k, "particles": n, "detections": nd, "landmarks": n_lm, "categories": n_cat, "steps": steps,
                "ms_per_step_e2e": mb, "member_steps_per_s": k * 1e3 / mb, "launches_per_step": int(max(launches)),
                "standalone_ms_per_round": ms, "standalone_member_steps_per_s": k * 1e3 / ms, "speedup": ms / mb, "kernels_ms": {},
                "device": device}
            batch.close()
            for a in singles:
                a.close()
    return res


def batch_reweight_ms(batch, poses, scans, steps):
    """Mean device time per step of the batch's reweight kernels (names containing batch_reweight or batch_beam), from
    torch.profiler in a run of its own; poses[t] and scans[t] are step t's inputs of every member."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(steps):
            batch.update(poses[t], scans[t])
    total_us = sum(e.device_time_total for e in prof.key_averages() if "batch_reweight" in e.key or "batch_beam" in e.key)
    return total_us / 1e3 / steps


def run_batch_maps():
    """K in {64, 256} members x 2000 particles x 100 points spread evenly (member m on map m % M) over M in {1, 4, 16}
    likelihood-field maps of 2000^2, each a different synthetic scene, systematic resampling, every member updating every
    step.  One AmclBatch with M maps against M single-map batches (K / M members each) stepped one after another, in the
    same process, alternating step by step.  Also the batch's reweight kernel time per step (torch.profiler, separate
    run), which shows what spreading the members' lookups over M tables (16 x 32 MB of fixed-point tables at M = 16,
    beyond the 50 MB L2) costs; and one mixed step (likelihood-field and beam members) with its launch count."""
    res = {}
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    n, steps, warmup = 2000, 20, 3
    device = device_record()
    scenes = [synthetic.make_scenario(grid_size=2000, n_beams=100, steps=warmup + steps, map_seed=42 + j) for j in range(16)]
    grids = [bb.OccupancyGrid(s.cells, s.resolution) for s in scenes]

    def make(members, maps):
        """A batch whose member i reads maps[i % len(maps)] (scene indices), initialised on that scene."""
        params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in members]
        b = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in members], params)
        ids = [b.add_likelihood_field_map(lfm, grids[j]) for j in maps]
        for i in range(len(members)):
            b.update_map(i, ids[i % len(maps)])
            s = scenes[maps[i % len(maps)]]
            b.initialize(i, s.initial_mean, s.initial_cov)
        return b

    def inputs(members, maps, t):
        return ([bb.se2(*scenes[maps[i % len(maps)]].poses[t]) for i in range(len(members))],
                [scenes[maps[i % len(maps)]].scans[t] for i in range(len(members))])

    for k in (64, 256):
        for n_maps in (1, 4, 16):
            maps = list(range(n_maps))
            multi = make(list(range(k)), maps)
            singles = [make(list(range(j, k, n_maps)), [j]) for j in maps]
            wall_multi, wall_singles, launches = [], [], []
            for t in range(warmup + steps):
                # both arms' inputs are built before their timed windows, which hold only the update calls
                poses, scans = inputs(range(k), maps, t)
                single_inputs = [inputs(range(j, k, n_maps), [j], t) for j in maps]
                before = multi.launch_count()
                t0 = time.perf_counter()
                r = multi.update(poses, scans)
                t1 = time.perf_counter()
                rs = [b.update(p, s) for b, (p, s) in zip(singles, single_inputs)]
                t2 = time.perf_counter()
                launches.append(multi.launch_count() - before)
                assert all(x.updated for x in r) and all(x.updated for rr in rs for x in rr)
                if t >= warmup:
                    wall_multi.append((t1 - t0) * 1e3)
                    wall_singles.append((t2 - t1) * 1e3)
            mb, ms = float(np.median(wall_multi)), float(np.median(wall_singles))
            prof_poses, prof_scans = zip(*[inputs(range(k), maps, t % (warmup + steps)) for t in range(10)])
            res[f"batch_maps_{k}_x_{n}_x_100_lfm_2000_{n_maps}_maps"] = {
                "members": k, "particles": n, "points": 100, "maps": n_maps, "steps": steps,
                "ms_per_step_e2e": mb, "member_steps_per_s": k * 1e3 / mb, "launches_per_step": int(max(launches)),
                "single_map_batches_ms_per_round": ms, "single_map_batches_member_steps_per_s": k * 1e3 / ms,
                "reweight_kernel_ms_per_step": batch_reweight_ms(multi, prof_poses, prof_scans, 10),
                "kernels_ms": {}, "device": device}
            del multi, singles
    # one mixed step: half the members on a likelihood field, half on a beam map of the same scene (two-pass walk)
    k = 64
    params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
    mixed = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)], params)
    ids = [mixed.add_likelihood_field_map(lfm, grids[0]), mixed.add_beam_map(bb.BeamModelParam(beam_max_range=60.0), grids[0])]
    for m in range(k):
        mixed.update_map(m, ids[m % 2])
        mixed.initialize(m, scenes[0].initial_mean, scenes[0].initial_cov)
    wall, launches = [], []
    for t in range(warmup + steps):
        pose = bb.se2(*scenes[0].poses[t])
        t0 = time.perf_counter()
        before = mixed.launch_count()
        assert all(x.updated for x in mixed.update([pose] * k, [scenes[0].scans[t]] * k))
        t1 = time.perf_counter()
        launches.append(mixed.launch_count() - before)
        if t >= warmup:
            wall.append((t1 - t0) * 1e3)
    mb = float(np.median(wall))
    res[f"batch_maps_mixed_{k}_x_{n}_x_100_lfm_and_beam_2000"] = {
        "members": k, "particles": n, "points": 100, "maps": 2, "steps": steps, "ms_per_step_e2e": mb,
        "member_steps_per_s": k * 1e3 / mb, "launches_per_step": int(max(launches)), "kernels_ms": {}, "device": device}
    return res


def select_host_ms(states, weights, repeats=50):
    """Host time of the select_cluster pass alone (bb200_cluster_select_host) on the cells of one member's particles at the
    default clusterizer parameters; the records come from a standalone filter's device histogram."""
    import ctypes as C

    from beluga_b200 import _capi

    lib = _capi.load()
    f = bb.Filter(capacity=len(states))
    f.set_particles(states, weights)
    n_bins, top = C.c_uint64(0), C.c_double(0.0)
    lib.bb200_filter_particle_histogram(f._h, 0.20, 0.524, None, 0, C.byref(n_bins), C.byref(top))
    m = n_bins.value
    cells = (_capi.ClusterCell * max(m, 1))()
    assert lib.bb200_filter_particle_histogram(f._h, 0.20, 0.524, cells, m, C.byref(n_bins), C.byref(top)) == 0
    p = _capi.ClusterParam(0.20, 0.524, 0.90)
    ids = (C.c_uint32 * max(m, 1))()
    n_clusters, found, best = C.c_uint32(0), C.c_int(0), C.c_uint32(0)
    out = np.zeros(9)
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        lib.bb200_cluster_select_host(cells, m, len(states), C.byref(p), ids, C.byref(n_clusters), C.byref(found), C.byref(best),
                                      out.ctypes.data_as(C.POINTER(C.c_double)))
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times)), m


def run_batch_cluster():
    """The `batch` workload (K in {1, 16, 64, 256} members x 2000 particles x 100 points, 2000^2 map, systematic resampling, every
    member updating every step) and K = 1 x 32 768 particles, timed as beluga_ros-shaped rounds: update, then the cluster-based
    estimate of every member, once as one cluster_estimates call and once as K cluster_estimate(m) calls, on the same particles.
    On a build without AmclBatch.cluster_estimates only the per-member form is timed."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    steps, warmup = 20, 3
    batched = hasattr(bb.AmclBatch, "cluster_estimates")
    device = device_record()
    for k, n in ((1, 2000), (16, 2000), (64, 2000), (256, 2000), (1, 32768)):
        params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)], params)
        batch.set_likelihood_field_map(lfm, grid)
        for m in range(k):
            batch.initialize(m, sc.initial_mean, sc.initial_cov)
        update_ms, all_ms, each_ms, all_launches, each_launches = [], [], [], [], []
        for t in range(warmup + steps):
            pose = bb.se2(*sc.poses[t])
            t0 = time.perf_counter()
            r = batch.update([pose] * k, [sc.scans[t]] * k)
            t1 = time.perf_counter()
            assert all(x.updated for x in r)
            if batched:
                before = batch.launch_count()
                t2 = time.perf_counter()
                together = batch.cluster_estimates()
                t3 = time.perf_counter()
                all_launches.append(batch.launch_count() - before)
            before = batch.launch_count()
            t4 = time.perf_counter()
            each = [batch.cluster_estimate(m) for m in range(k)]
            t5 = time.perf_counter()
            each_launches.append(batch.launch_count() - before)
            if batched:
                assert all(a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() for a, b in zip(together, each))
            if t >= warmup:
                update_ms.append((t1 - t0) * 1e3)
                each_ms.append((t5 - t4) * 1e3)
                if batched:
                    all_ms.append((t3 - t2) * 1e3)
        states, weights = batch.particles(0)
        select_ms, cells = select_host_ms(states, weights)
        row = {"members": k, "particles": n, "points": 100, "steps": steps, "update_ms": float(np.median(update_ms)),
               "per_member_estimates_ms": float(np.median(each_ms)),
               "round_ms_per_member_form": float(np.median(np.add(update_ms, each_ms))),
               "launches_per_member_call": int(max(each_launches)) / k,
               "select_cluster_host_ms_one_member": select_ms, "cells_member_0": cells,
               "ms_per_step_e2e": float(np.median(np.add(update_ms, all_ms if batched else each_ms))), "kernels_ms": {}, "device": device}
        if batched:
            row.update({"batched_estimates_ms": float(np.median(all_ms)), "round_ms_batched_form": float(np.median(np.add(update_ms, all_ms))),
                        "launches_per_batched_call": int(max(all_launches))})
        res[f"batch_cluster_{k}_x_{n}_x_100_lfm_2000"] = row
    return res


def run_batch_clustered():
    """One beluga_ros node cycle for every member, two ways, on the `batch_cluster` shapes (K in {1, 16, 64, 256} members x
    2000 particles x 100 points on the 2000^2 map, and K = 1 x 32 768): update_clustered (the update and every updated
    member's cluster-based estimate in one call, the per-cell flood on the device) against update_measurements followed by
    cluster_estimates (the flood on the host, member after member).  Two batches built alike take the same inputs; the two
    forms alternate which goes first from round to round, and their results and estimates are compared byte for byte."""
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    steps, warmup = 20, 3
    device = device_record()
    for k, n in ((1, 2000), (16, 2000), (64, 2000), (256, 2000), (1, 32768)):
        params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
        batches = {}
        for form in ("clustered", "separate"):
            batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)], params)
            batch.set_likelihood_field_map(lfm, grid)
            for m in range(k):
                batch.initialize(m, sc.initial_mean, sc.initial_cov)
            batches[form] = batch
        times = {"clustered": [], "separate": []}
        launches = {"clustered": [], "separate": []}
        for t in range(warmup + steps):
            pose = bb.se2(*sc.poses[t])
            out = {}
            for form in (("clustered", "separate") if t % 2 == 0 else ("separate", "clustered")):
                batch = batches[form]
                before = batch.launch_count()
                t0 = time.perf_counter()
                if form == "clustered":
                    out[form] = batch.update_clustered([pose] * k, [sc.scans[t]] * k)
                else:
                    r = batch.update_measurements([pose] * k, [sc.scans[t]] * k)
                    out[form] = (r, batch.cluster_estimates(present=[bool(x.updated) for x in r]))
                t1 = time.perf_counter()
                launches[form].append(batch.launch_count() - before)
                if t >= warmup:
                    times[form].append((t1 - t0) * 1e3)
            for a, b in zip(out["clustered"][1], out["separate"][1]):
                assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        row = {"members": k, "particles": n, "points": 100, "steps": steps, "device": device, "kernels_ms": {},
               "ms_per_step_e2e": float(np.median(times["clustered"]))}
        for form in times:
            row[f"{form}_round_ms_median"] = float(np.median(times[form]))
            row[f"{form}_round_ms_range"] = [float(np.min(times[form])), float(np.max(times[form]))]
            row[f"{form}_launches_per_round"] = int(max(launches[form]))
        row["speedup_median"] = row["separate_round_ms_median"] / row["clustered_round_ms_median"]
        res[f"batch_clustered_{k}_x_{n}_x_100_lfm_2000"] = row
    return res


def run_batch_cloud():
    """The `batch` workload (K in {1, 16, 64, 256} members x 2000 particles x 100 points, 2000^2 map, systematic resampling)
    and K standalone Amcl fed the same inputs, timed as one particle-cloud publish round after each update: the batched form
    is one particle_histograms call and one sample_states call of 2000 poses per member; the per-node form is each standalone
    filter's particle_histogram and sample_states in turn.  The two forms alternate which goes first from round to round,
    their outputs are compared byte for byte, and the host marker geometry (bb200_particle_cloud_markers over every member's
    bins) is timed on its own."""
    import ctypes as C

    from beluga_b200 import _capi

    lib = _capi.load()
    res = {}
    sc = synthetic.make_scenario(grid_size=2000, n_beams=100, steps=100)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    steps, warmup, n = 20, 3, 2000
    device = device_record()
    for k in (1, 16, 64, 256):
        params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
        motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
        batch = bb.AmclBatch(motions, params)
        batch.set_likelihood_field_map(lfm, grid)
        nodes = []
        for m in range(k):
            batch.initialize(m, sc.initial_mean, sc.initial_cov)
            a = bb.Amcl(motions[m], params[m])
            a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid)
            a.initialize(sc.initial_mean, sc.initial_cov)
            nodes.append(a)
        batched_ms, node_ms, markers_ms, batched_launches = [], [], [], []
        for t in range(warmup + steps):
            pose = bb.se2(*sc.poses[t])
            assert all(x.updated for x in batch.update([pose] * k, [sc.scans[t]] * k))
            for a in nodes:
                a.update(pose, sc.scans[t])
            step = 0xFFFFFFFF - t

            def batched():
                before = batch.launch_count()
                t0 = time.perf_counter()
                hists = batch.particle_histograms()
                poses = batch.sample_states(n, step)
                t1 = time.perf_counter()
                batched_launches.append(batch.launch_count() - before)
                return (t1 - t0) * 1e3, hists, poses

            def per_node():
                t0 = time.perf_counter()
                out = [(a.filter.particle_histogram(), a.filter.sample_states(n, step)) for a in nodes]
                return (time.perf_counter() - t0) * 1e3, out

            if t % 2 == 0:
                b_ms, hists, poses = batched()
                p_ms, each = per_node()
            else:
                p_ms, each = per_node()
                b_ms, hists, poses = batched()
            for m in range(k):
                (rep, w, _, _, top), s = each[m]
                assert hists[m][0]["rep"].tobytes() == rep.tobytes() and hists[m][0]["weight"].tobytes() == w.tobytes()
                assert hists[m][1] == top and poses[m].tobytes() == s.tobytes()
            t0 = time.perf_counter()
            for bins, _ in hists:
                cells = bins.ctypes.data_as(C.POINTER(_capi.ClusterCell))
                bodies, heads = (_capi.MarkerVertex * (2 * len(bins)))(), (_capi.MarkerVertex * (3 * len(bins)))()
                scale = C.c_double(0.0)
                assert lib.bb200_particle_cloud_markers(cells, len(bins), bodies, heads, C.byref(scale)) == 0
            t1 = time.perf_counter()
            if t >= warmup:
                batched_ms.append(b_ms)
                node_ms.append(p_ms)
                markers_ms.append((t1 - t0) * 1e3)
        res[f"batch_cloud_{k}_x_{n}_x_100_lfm_2000"] = {
            "members": k, "particles": n, "points": 100, "samples_per_member": n, "steps": steps,
            "batched_publish_ms": float(np.median(batched_ms)), "batched_publish_ms_min_max": [float(np.min(batched_ms)), float(np.max(batched_ms))],
            "per_node_publish_ms": float(np.median(node_ms)), "per_node_publish_ms_min_max": [float(np.min(node_ms)), float(np.max(node_ms))],
            "host_marker_geometry_ms": float(np.median(markers_ms)), "launches_per_batched_round": int(max(batched_launches)),
            "ms_per_step_e2e": float(np.median(batched_ms)), "kernels_ms": {}, "device": device}
    return res


def run_batch_measurements():
    """AmclBatch fed sensor messages: K in {1, 16, 64, 256} members x 2000 particles with {100, 1080}-beam laser scans, and 16
    members with 64 x 1024 = 65 536-point lidar clouds, on the 2000^2 synthetic map.  Two batches step the same members in
    turn: one with bb200_amcl_batch_update_measurements (scans and clouds converted on the device), one with K calls of
    bb200_scan_to_points / bb200_point_cloud_to_points and bb200_amcl_batch_update.  The ctypes arguments of every step
    are built before the timing, so each time is the C calls alone, end to end (median of 20 steps)."""
    import ctypes as C

    from beluga_b200 import _capi

    lib = _capi.load()
    res = {}
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    n, steps, warmup = 2000, 20, 3
    device = device_record()
    cases = [("scan", k, beams) for beams in (100, 1080) for k in (1, 16, 64, 256)] + [("cloud", 16, 65_536)]
    scenes = {}
    for kind, k, size in cases:
        key = 1080 if kind == "cloud" else size
        if key not in scenes:
            scenes[key] = synthetic.make_scenario(grid_size=2000, n_beams=key, steps=warmup + steps + 1)
        sc = scenes[key]
        grid = bb.OccupancyGrid(sc.cells, sc.resolution)
        params = [bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=m) for m in range(k)]
        motions = [bb.DifferentialDriveModelParam(*MOTION) for _ in range(k)]
        batches = {}
        for form in ("device", "host"):
            b = bb.AmclBatch(motions, params)
            b.set_likelihood_field_map(lfm, grid)
            for m in range(k):
                b.initialize(m, sc.initial_mean, sc.initial_cov)
            batches[form] = b
        # Every step's messages, one per member (the members of a step share the scene's message).
        msgs, keep = [], []
        for t in range(warmup + steps):
            if kind == "scan":
                r = np.hypot(*sc.scans[t].T).astype(np.float32)
                m, kept = bb._laser_scan(r, np.float32(-np.pi), np.float32(2 * np.pi / size), 0.0, float("inf"), 0, None)
                meas = _capi.Measurement(_capi.MEASUREMENT_SCAN, None, 0, C.pointer(m), None)
            else:
                pc = synthetic.make_point_cloud(sc, t, rows=64, azimuths=1024)
                m, kept = bb._point_cloud(pc.data, pc.point_step, pc.x_offset, pc.datatype, pc.origin, None)
                meas = _capi.Measurement(_capi.MEASUREMENT_CLOUD, None, 0, None, C.pointer(m))
            msgs.append((m, (_capi.Measurement * k)(*([meas] * k)), bb.se2(*sc.poses[t])))
            keep.append(kept)
        bufs = [np.zeros((size + 1, 2)) for _ in range(k)]
        ptrs = (C.POINTER(C.c_double) * k)(*[b.ctypes.data_as(C.POINTER(C.c_double)) for b in bufs])
        counts = (C.c_uint64 * k)()
        results = (_capi.UpdateResult * k)()
        wall = {"device": [], "host": []}
        launches = []
        for t, (m, table, pose) in enumerate(msgs):
            poses = np.tile(pose, (k, 1))
            pp = poses.ctypes.data_as(C.POINTER(C.c_double))
            before = batches["device"].launch_count()
            t0 = time.perf_counter()
            assert lib.bb200_amcl_batch_update_measurements(batches["device"]._h, pp, table, None, results) == 0
            t1 = time.perf_counter()
            launches.append(batches["device"].launch_count() - before)
            assert all(x.updated for x in results)
            cn = C.c_uint64()
            for j in range(k):
                if kind == "scan":
                    assert lib.bb200_scan_to_points(C.byref(m), ptrs[j], size + 1, C.byref(cn)) == 0
                else:
                    assert lib.bb200_point_cloud_to_points(C.byref(m), ptrs[j], size + 1, C.byref(cn)) == 0
                counts[j] = cn.value
            assert lib.bb200_amcl_batch_update(batches["host"]._h, pp, ptrs, counts, None, results) == 0
            t2 = time.perf_counter()
            if t >= warmup:
                wall["device"].append((t1 - t0) * 1e3)
                wall["host"].append((t2 - t1) * 1e3)
        md, mh = float(np.median(wall["device"])), float(np.median(wall["host"]))
        per_point = 4 if kind == "scan" else 12
        res[f"batch_measurements_{kind}_{k}_x_{n}_x_{size}_lfm_2000"] = {
            "members": k, "particles": n, "kind": kind, "points": size, "steps": steps,
            "ms_per_step_e2e": md, "ms_per_step_e2e_min_max": [float(np.min(wall["device"])), float(np.max(wall["device"]))],
            "host_converted_ms_per_step": mh, "host_converted_ms_min_max": [float(np.min(wall["host"])), float(np.max(wall["host"]))],
            "upload_bytes_per_member": per_point * size, "host_converted_upload_bytes_per_member": 16 * size,
            "launches_per_step": int(max(launches)), "kernels_ms": {}, "device": device}
    return res


def main():
    out = {}
    which = sys.argv[1:] or ["c1", "c3", "c4"]
    if "c1" in which:
        sc = synthetic.make_scenario(grid_size=500, n_beams=180, steps=100)
        n = 10_000
        res = run_gpu(sc, bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM),
                      bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_MULTINOMIAL, seed=1), steps=20)
        from oracle import pyoracle as orc

        for threads, tag in ((1, "cpu_seq"), (min(os.cpu_count() or 1, 16), "cpu_par")):
            o = orc.Amcl(orc.AmclParam(min_particles=n, max_particles=n, scheme=0, seed=1, rng_mode=1, threads=threads), orc.MotionParam(*MOTION))
            o.set_map(0, orc.LfmParam(**LFM), orc.Grid(sc.cells, sc.resolution))
            o.initialize_normal(sc.initial_mean, sc.initial_cov)
            o.update(orc.se2(*sc.poses[0]), sc.scans[0])
            t0 = time.perf_counter()
            for k in range(1, 11):
                o.update(orc.se2(*sc.poses[k]), sc.scans[k])
            res[tag + "_ms_per_step"] = (time.perf_counter() - t0) / 10 * 1e3
            res[tag + "_threads"] = threads
        out["c1_10k_x_180_lfm_500_multinomial"] = res
    if "c3" in which:
        from oracle import pyoracle as orc

        sc = synthetic.make_scenario(grid_size=2000, n_beams=720, steps=100)
        n = 1_000_000
        res = run_gpu(sc, bb.SENSOR_BEAM, bb.BeamModelParam(beam_max_range=60.0),
                      bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1), steps=5, warmup=1)
        # L-bar (cells the reference's Bresenham walk inspects per beam) and the CPU port on a posterior-like sample
        rng = np.random.default_rng(3)
        m = 4000
        pose = sc.poses[3]
        st = np.array([orc.se2(pose[0] + rng.normal(0, 0.3), pose[1] + rng.normal(0, 0.3), pose[2] + rng.normal(0, 0.25)) for _ in range(m)])
        orc.use_native_build()
        bp = orc.BeamParam(beam_max_range=60.0)
        t0 = time.perf_counter()
        _, visited = orc.sensor_weights(orc.BEAM, bp, orc.Grid(sc.cells, sc.resolution), sc.scans[3], st, return_visited=True)
        cpu_s = time.perf_counter() - t0
        lbar = visited / (m * 720)
        k = res["kernels_ms"].get("reweight_beam", float("nan"))
        # SURVEY 8(d): A = N * (48 + B * L-bar) bytes for the reweight launch (one occupancy byte per inspected cell)
        a_bytes = n * (48 + 720 * lbar)
        res.update({"cells_per_ray_reference": lbar, "algorithmic_bytes_reweight": a_bytes,
                    "reweight_achieved_gbs": a_bytes / (k * 1e-3) / 1e9,
                    "cpu_reweight_ms_per_1M_particles": cpu_s * 1e3 * n / m, "cpu_sample": f"{m} particles x 720 beams, all OpenMP threads, scaled x{n // m} (extrapolated)"})
        out["c3_1M_x_720_beam_2000"] = res
    if "c4" in which:
        sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=100)
        out["c4_kld_100k_10M_lfm"] = run_gpu(sc, bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM),
                                             bb.AmclParams(min_particles=100_000, max_particles=10_000_000, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1,
                                                           spatial_resolution=(0.5, 0.5, float(np.deg2rad(10.0)))), steps=6, warmup=1)  # beluga_ros defaults (SURVEY 8d)
    if "cloud" in which:
        out.update(run_cloud())
    if "batch" in which:
        out.update(run_batch())
    if "batch_kld" in which:
        out.update(run_batch_kld())
    if "batch_selective" in which:
        out.update(run_batch_selective())
    if "batch_cluster" in which:
        out.update(run_batch_cluster())
    if "batch_clustered" in which:
        out.update(run_batch_clustered())
    if "batch_cloud" in which:
        out.update(run_batch_cloud())
    if "batch_members" in which:
        out.update(run_batch_members())
    if "batch_state" in which:
        out.update(run_batch_state())
    if "batch_beam" in which:
        out.update(run_batch_beam())
    if "batch_maps" in which:
        out.update(run_batch_maps())
    if "batch_measurements" in which:
        out.update(run_batch_measurements())
    if "raycast" in which:
        out.update(run_raycast())
    if "weighed" in which:
        out.update(run_weighed())
    if "sharded-publish" in which:
        out.update(run_sharded_publish())
    if "sharded-weighed" in which:
        out.update(run_sharded_weighed())
    if "landmark" in which:
        out.update(run_landmark())
    if "batch_landmark" in which:
        out.update(run_batch_landmark())
    if "sharded_landmark" in which:
        out.update(run_sharded_landmark())
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    path = os.path.join(ROOT, "gpurun_out", "configs.json")
    merged = json.load(open(path)) if os.path.exists(path) else {}
    tag = os.environ.get("BB200_CONFIG_TAG", "")
    merged.update({k + tag: v for k, v in out.items()})
    json.dump(merged, open(path, "w"), indent=1)
    for k, v in out.items():
        print(k + tag, "e2e ms/step", round(v["ms_per_step_e2e"], 3), "kernels", v["kernels_ms"])


if __name__ == "__main__":
    main()
