#!/usr/bin/env python
"""Headless driver with the reference's CLI (`run_simulation.py --scene_file ...`,
reference run_simulation.py:11-35,79-112) on top of the CUDA engine.

The GGUI window / camera / PNG export of the reference are out of scope; the simulation loop, the
`numberOfStepsPerRenderUpdate` substepping, the `output_interval = int(0.016 / dt)` cadence and
the ASCII PLY export of object 0 (`exportPly`) are kept.  Extra flags: --frames, --quiet, --gpus.

`--gpus N` runs the scene x-slab sharded (sph_taichi_b200.slab) across N GPUs of a node, one process per GPU:

    python -m torch.distributed.run --nproc-per-node N run_simulation.py --scene dragon_bath --gpus N

The loop and the output files are those of the single-GPU run; rank 0 writes them (`ShardedSimulation.dump`
gathers object 0 over the engine's own transport; the torch process group, gloo, only carries the NCCL id).
`--gpus 1` runs the sharded engine on one GPU without torch.distributed.run.  IISPH scenes (simulationMethod 3) shard
only on request, `--gpus N --shard-iisph`; without the flag they are refused.  IISPH scenes with dynamic solids need
`--gpus N --shard-iisph-bodies` (which implies `--shard-iisph`).
"""
import argparse
import copy
import os
import time

import numpy as np

from sph_taichi_b200 import ParticleSystem, SimConfig


def write_ply_ascii(path, pos):
    with open(path, "w") as fh:
        # header as ti.tools.PLYWriter.export_frame_ascii prints it (comment line included; restated from the
        # Taichi docs, the wheel is not installable offline)
        fh.write("ply\nformat ascii 1.0\ncomment created by PLYWriter\n")
        fh.write(f"element vertex {pos.shape[0]}\nproperty float x\nproperty float y\nproperty float z\nend_header\n")
        np.savetxt(fh, pos, fmt="%.7g")


def write_obj(path, verts, faces):
    with open(path, "w") as f:
        for v in verts:
            f.write(f"v {v[0]:.7g} {v[1]:.7g} {v[2]:.7g}\n")
        for t in faces:
            f.write(f"f {t[0] + 1} {t[1] + 1} {t[2] + 1}\n")


def run_single(config, scene_name, frames, quiet=False):
    """The single-GPU run: `frames` render updates of the reference's loop with its exports."""
    substeps = config.get_cfg("numberOfStepsPerRenderUpdate")
    output_interval = int(0.016 / config.get_cfg("timeStepSize"))
    output_ply = config.get_cfg("exportPly")
    output_obj = config.get_cfg("exportObj")
    series_prefix = "{}_output/particle_object_{}.ply".format(scene_name, "{}")
    if output_ply or output_obj:
        os.makedirs(f"{scene_name}_output", exist_ok=True)

    ps = ParticleSystem(config, GGUI=False)
    solver = ps.build_solver()
    solver.initialize()

    cnt = 0
    cnt_ply = 0
    t0 = time.perf_counter()
    while cnt < frames:
        solver.step(substeps)
        if cnt % output_interval == 0 and output_ply:
            obj_data = ps.dump(obj_id=0)
            write_ply_ascii(series_prefix.format(0).replace(".ply", f"_{cnt_ply:06}.ply"), obj_data["position"])
        if cnt % output_interval == 0 and output_obj:
            # posed rigid meshes (reference run_simulation.py:108-111); needs the mesh files on disk
            for r_body_id in ps.object_id_rigid_body:
                obj = ps.object_collection[r_body_id]
                if "meshFaces" not in obj:
                    continue
                verts = obj.get("meshVertices", obj["restPosition"])
                write_obj(f"{scene_name}_output/obj_{r_body_id}_{cnt_ply:06}.obj", verts, obj["meshFaces"])
        if cnt % output_interval == 0 and (output_ply or output_obj):
            cnt_ply += 1
        cnt += 1
    ps._engine.check_status()
    dt = time.perf_counter() - t0
    if not quiet:
        print(f"{scene_name}: {ps.particle_max_num} particles, {cnt * substeps} steps in {dt:.3f} s "
              f"({cnt * substeps / dt:.1f} steps/s incl. exports)")
    return 0


def _resolved_scene(config):
    """The scene as a dict whose mesh / fixture paths resolve from any working directory (build_sharded reads a
    dict; the single engine looks the files up relative to the scene file's directory too)."""
    sc = copy.deepcopy(config.config)
    for body in sc.get("RigidBodies", []):
        for key, cands in (("geometryFile", lambda p: [p, os.path.join(config.scene_dir, p),
                                                       os.path.join(config.scene_dir, "..", "..", p)]),
                           ("voxelizedPointsFile", lambda p: [p, os.path.join(config.scene_dir, p)])):
            if body.get(key):
                found = [p for p in cands(body[key]) if os.path.isfile(p)]
                if found:
                    body[key] = os.path.abspath(found[0])
    return sc


def run_sharded(config, scene_name, frames, device, transport=None, quiet=False, iisph=False, iisph_bodies=False):
    """The same loop and output files as `run_single`, on the x-slab sharded engine: this process is rank RANK of
    WORLD_SIZE (environment, default 0 of 1) on `device`.  Every rank steps and joins each `dump`; rank 0 writes the
    files and prints the summary.  `transport`: an SphTransport object in place of the library's NCCL communicator
    (slab.GlooTransport); with world > 1 and no transport the torch process group must be initialised.  `iisph`:
    shard an IISPH scene (`slab.build_sharded(..., iisph=True)`); `iisph_bodies`: one with dynamic solids
    (`iisph_bodies=True`)."""
    from sph_taichi_b200 import slab
    from sph_taichi_b200.sph_base import posed_mesh

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    try:
        sim, n_total = slab.build_sharded(_resolved_scene(config), rank, world, device, transport=transport,
                                          dynamic_solids=slab.scene_has_dynamic_solids(config), iisph=iisph,
                                          iisph_bodies=iisph_bodies)
    except NotImplementedError as exc:
        raise SystemExit(f"{scene_name}: {exc}") from exc
    substeps = config.get_cfg("numberOfStepsPerRenderUpdate")
    output_interval = int(0.016 / config.get_cfg("timeStepSize"))
    output_ply = config.get_cfg("exportPly")
    output_obj = config.get_cfg("exportObj")
    series_prefix = "{}_output/particle_object_{}.ply".format(scene_name, "{}")
    if rank == 0 and (output_ply or output_obj):
        os.makedirs(f"{scene_name}_output", exist_ok=True)
    body_index = {oid: b for b, (oid, *_rest) in enumerate(sim.bodies or [])}

    cnt = 0
    cnt_ply = 0
    t0 = time.perf_counter()
    while cnt < frames:
        sim.step(substeps)
        if cnt % output_interval == 0 and output_ply:
            obj_data = sim.dump(0)  # collective
            if rank == 0:
                write_ply_ascii(series_prefix.format(0).replace(".ply", f"_{cnt_ply:06}.ply"), obj_data["position"])
        if cnt % output_interval == 0 and output_obj and rank == 0:
            # cm and R of a body are bit-identical on every rank; bodies that are not shape-matched keep their rest pose
            for oid, obj in sim.object_collection.items():
                if "meshFaces" not in obj:
                    continue
                verts = obj["restPosition"]
                if oid in body_index:
                    cm, R = sim.body_state(body_index[oid])
                    verts = posed_mesh(obj["restPosition"], obj["restCenterOfMass"], R, cm)
                write_obj(f"{scene_name}_output/obj_{oid}_{cnt_ply:06}.obj", verts, obj["meshFaces"])
        if cnt % output_interval == 0 and (output_ply or output_obj):
            cnt_ply += 1
        cnt += 1
    sim.info()  # raises on a capacity / out-of-grid flag
    dt = time.perf_counter() - t0
    if rank == 0 and not quiet:
        print(f"{scene_name}: {n_total} particles, {cnt * substeps} steps in {dt:.3f} s "
              f"({cnt * substeps / dt:.1f} steps/s incl. exports) on {world} GPUs")
    return 0


def main_sharded(args, config, scene_name):
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} needs WORLD_SIZE={args.gpus} (launch with torch.distributed.run); "
                         f"got WORLD_SIZE={world}")
    dev = torch.device(f"cuda:{local}")
    torch.cuda.set_device(dev)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        dist.init_process_group("gloo", rank=rank, world_size=world)  # carries the NCCL id only
    try:
        return run_sharded(config, scene_name, args.frames, dev, quiet=args.quiet, iisph=args.shard_iisph,
                           iisph_bodies=args.shard_iisph_bodies)
    finally:
        if world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description="SPH (CUDA engine)")
    parser.add_argument("--scene_file", default="", help="scene file (JSON, the reference's schema)")
    parser.add_argument("--scene", default="", help="built-in scene name instead of a file, e.g. dragon_bath "
                                                    "(python -m sph_taichi_b200.scene DIR writes them as JSON)")
    parser.add_argument("--frames", type=int, default=100, help="render updates to run (the reference loops until the window closes)")
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument("--gpus", type=int, default=None,
                        help="x-slab sharded run on N GPUs, one process per GPU (N > 1: under torch.distributed.run)")
    parser.add_argument("--shard-iisph", action="store_true",
                        help="with --gpus: shard an IISPH scene (simulationMethod 3; fluid and static solids)")
    parser.add_argument("--shard-iisph-bodies", action="store_true",
                        help="with --gpus: shard an IISPH scene with dynamic solids (implies --shard-iisph)")
    args = parser.parse_args()
    if args.shard_iisph_bodies and args.gpus is None:
        parser.error("--shard-iisph-bodies needs --gpus N")
    if args.shard_iisph and args.gpus is None:
        parser.error("--shard-iisph needs --gpus N")
    if args.scene:
        from sph_taichi_b200 import scene as _scene
        scene_path = args.scene + ".json"
        config = SimConfig(_scene.NAMED_SCENES[args.scene]())
    else:
        scene_path = args.scene_file
        config = SimConfig(scene_file_path=scene_path)
    scene_name = scene_path.split("/")[-1].split(".")[0]
    if args.gpus is None:
        run_single(config, scene_name, args.frames, quiet=args.quiet)
    else:
        raise SystemExit(main_sharded(args, config, scene_name))
