"""Worker of tests/test_gpu_sharded.py: one rank (one GPU) of a sharded filter; rank 0 also runs the
same filter on a single GPU and compares -- results must not depend on the number of ranks.

    python -m torch.distributed.run --nproc-per-node=R _shard_gpu_worker.py SHARD STEPS MODE

MODE: nccl, nccl-recovery, nccl-selective (NCCL collectives from Python), p2p, p2p-recovery, p2p-multinomial,
p2p-kld (the exchanges through peer memory inside the library)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import beluga_b200 as bb  # noqa: E402
from beluga_b200 import synthetic  # noqa: E402
from beluga_b200.distributed import ShardedAmcl  # noqa: E402


def main():
    local_rank = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    rank, world = dist.get_rank(), dist.get_world_size()
    shard, steps = int(sys.argv[1]), int(sys.argv[2])
    mode = sys.argv[3] if len(sys.argv) > 3 else "nccl"
    p2p = mode.startswith("p2p")
    scheme = bb.RESAMPLE_MULTINOMIAL if mode == "p2p-multinomial" else bb.RESAMPLE_SYSTEMATIC
    inject = 0.03 if mode.endswith("recovery") or mode == "p2p-multinomial" else None  # random_intersperse probability
    kld_min = 500 if mode == "p2p-kld" else None  # KLD-adaptive particle count on shards (peer-memory path)
    # every other step keeps its particles, the others resample only when the effective sample size drops
    selective = dict(selective_resampling=True, resample_interval=2) if mode == "nccl-selective" else {}
    total = shard * world
    sc = synthetic.make_scenario(grid_size=200, n_beams=181, steps=steps + 1)
    motion = bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05)
    lfm = bb.LikelihoodFieldModelParam(max_obstacle_distance=2.0, max_laser_distance=100.0)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)

    override = inject if (p2p and inject is not None) else 0.0  # the peer-memory path takes the injection probability as a parameter
    sharded = ShardedAmcl(motion, bb.AmclParams(resample_scheme=scheme, seed=21, device=local_rank, recovery_probability_override=override, **selective),
                          shard=shard, p2p=p2p, kld_min_particles=kld_min)
    sharded.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid)
    sharded.initialize(sc.initial_mean, sc.initial_cov)
    single = None
    if rank == 0:
        single = bb.Amcl(motion, bb.AmclParams(min_particles=kld_min or total, max_particles=total, resample_scheme=scheme, seed=21, device=0,
                                               recovery_probability_override=override, **selective))
        single.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid)
        single.initialize(sc.initial_mean, sc.initial_cov)

    resampled = []
    for k in range(steps):
        pose = bb.se2(*sc.poses[k])
        out = sharded.update(pose, sc.scans[k], random_state_probability=None if p2p else inject)
        assert out is not None
        mean, cov, info = out
        resampled.append(info["resampled"])
        # gather the sharded particle set on rank 0 (a KLD-sized filter holds fewer than `shard` particles per rank)
        states, weights = sharded.filter.particles()
        padded = np.zeros((shard, 4))
        padded[: len(states)] = states
        counts = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(world)]
        dist.all_gather(counts, torch.tensor([len(states)], dtype=torch.int64, device="cuda"))
        gathered = [torch.zeros(shard, 4, dtype=torch.float64, device="cuda") for _ in range(world)]
        dist.all_gather(gathered, torch.from_numpy(padded).cuda())
        gathered = [g[: int(c.item())] for g, c in zip(gathered, counts)]
        if selective:
            gathered_weights = [torch.zeros(shard, dtype=torch.float64, device="cuda") for _ in range(world)]
            dist.all_gather(gathered_weights, torch.from_numpy(weights).cuda())
        if rank == 0:
            if inject is None or p2p:
                r = single.update(pose, sc.scans[k])
                ref_sum, ref_mean, ref_cov = r.weight_sum, np.array(r.estimate.mean), np.array(r.estimate.cov).reshape(3, 3)
            else:  # the same step composed from the filter-level calls, with the injection probability forced
                plan = single.plan_update(pose)
                sf = single.filter
                sf.propagate_reweight(plan.sampling, plan.step, sc.scans[k])
                factor, _ = sf.normalize()
                ref_sum = factor
                sf.resample(scheme, plan.step, total, random_state_probability=inject)
                ref_mean, ref_cov = sf.estimate()
                single.commit_update(True, inject)
            ref_states, ref_w = single.particles()
            all_states = torch.cat(gathered).cpu().numpy()
            assert len(all_states) == len(ref_states) == info["n_particles"], f"step {k}: {len(all_states)} particles on shards, {len(ref_states)} on one GPU"
            assert np.array_equal(all_states, ref_states), f"step {k}: sharded particle set differs from the single-GPU one"
            if selective:  # a step that keeps its particles leaves them normalised weights
                assert info["resampled"] == bool(r.resampled), f"step {k}: the sharded filter decided otherwise whether to resample"
                all_weights = torch.cat(gathered_weights).cpu().numpy()
                assert np.array_equal(all_weights, ref_w), f"step {k}: sharded weights differ from the single-GPU ones"
            else:
                assert np.all(weights == 1.0) and np.all(ref_w == 1.0)
            assert info["weight_sum"] == ref_sum
            tol = 1e-11 if kld_min else 1e-12  # KLD: the single filter re-reads its new set for the estimate, the shards sum what they produced
            assert np.abs(mean - ref_mean).max() < tol
            assert np.abs(cov - ref_cov).max() < tol
    if selective:
        assert any(resampled) and not all(resampled), f"selective resampling should both resample and keep: {resampled}"
    sharded.close()
    dist.barrier()
    if rank == 0:
        print("SHARD_GPU_WORKER_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
