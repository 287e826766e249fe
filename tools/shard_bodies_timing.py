"""Timing of the sharded WCSPH step with dynamic solids (build_sharded(dynamic_solids=True)) against the plain engine
on rank 0's GPU, in the same run.  Runs under torchrun (one rank per GPU) or as a plain world-1 process:

    python tools/shard_bodies_timing.py --scene armadillo_bath_dynamic --steps 100 --warm 30
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29541 \
        tools/shard_bodies_timing.py --scene armadillo_bath_dynamic

CUDA events around `--steps` steps after `--warm` warm-up steps; ms_per_step is the slowest rank's.  Prints one JSON
line with the card's name and power limit.
"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
from sph_taichi_b200 import ParticleSystem, SimConfig, scene, slab

ap = argparse.ArgumentParser()
ap.add_argument("--scene", default="armadillo_bath_dynamic")
ap.add_argument("--steps", type=int, default=100)
ap.add_argument("--warm", type=int, default=30)
a = ap.parse_args()
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", rank))
dev = torch.device(f"cuda:{local}")
torch.cuda.set_device(dev)
if world > 1:
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)


def timed(step, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(); step(k); e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


sc = scene.NAMED_SCENES[a.scene]()
sim, n_total = slab.build_sharded(sc, rank, world, dev, dynamic_solids=True)
sim.step(a.warm)
if world > 1:
    dist.barrier()
ms = torch.tensor([timed(sim.step, a.steps)], device=dev)
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
sim.info()  # raises on a status flag
launches0 = sim.launch_count(); sim.step(1); launches = sim.launch_count() - launches0
sim.eng.close()
del sim
torch.cuda.empty_cache()
if rank == 0:
    ps = ParticleSystem(SimConfig(sc), device=dev)
    solver = ps.build_solver(); solver.initialize()
    solver.step(a.warm)
    plain = timed(solver.step, a.steps)
    card, plimit = slab._gpu_name_and_power_limit(local)
    print(json.dumps({"scene": a.scene, "particles": int(n_total), "world": world, "steps": a.steps, "warm": a.warm,
                      "ms_per_step_sharded": round(float(ms.item()), 4), "ms_per_step_plain_rank0": round(plain, 4),
                      "slowdown_vs_plain": round(float(ms.item()) / plain, 3), "kernels_per_step_sharded": launches,
                      "gpu": card, "power_limit_w": plimit,
                      "note": "CUDA events around the timed steps after warm-up; sharded: eager launches, the slowest "
                              "rank; plain: the single engine's CUDA-graph step on rank 0's GPU, same run"}), flush=True)
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
