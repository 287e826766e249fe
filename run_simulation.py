#!/usr/bin/env python
"""Headless driver with the reference's CLI (`run_simulation.py --scene_file ...`,
reference run_simulation.py:11-35,79-112) on top of the CUDA engine.

The GGUI window / camera / PNG export of the reference are out of scope; the simulation loop, the
`numberOfStepsPerRenderUpdate` substepping, the `output_interval = int(0.016 / dt)` cadence and
the ASCII PLY export of object 0 (`exportPly`) are kept.  Extra flags: --frames, --quiet.
"""
import argparse
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


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description="SPH (CUDA engine)")
    parser.add_argument("--scene_file", default="", help="scene file (JSON, the reference's schema)")
    parser.add_argument("--scene", default="", help="built-in scene name instead of a file, e.g. dragon_bath "
                                                    "(python -m sph_taichi_b200.scene DIR writes them as JSON)")
    parser.add_argument("--frames", type=int, default=100, help="render updates to run (the reference loops until the window closes)")
    parser.add_argument("--quiet", action="store_true")
    args = parser.parse_args()
    if args.scene:
        from sph_taichi_b200 import scene as _scene
        scene_path = args.scene + ".json"
        config = SimConfig(_scene.NAMED_SCENES[args.scene]())
    else:
        scene_path = args.scene_file
        config = SimConfig(scene_file_path=scene_path)
    scene_name = scene_path.split("/")[-1].split(".")[0]

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
    while cnt < args.frames:
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
                with open(f"{scene_name}_output/obj_{r_body_id}_{cnt_ply:06}.obj", "w") as f:
                    for v in verts:
                        f.write(f"v {v[0]:.7g} {v[1]:.7g} {v[2]:.7g}\n")
                    for t in obj["meshFaces"]:
                        f.write(f"f {t[0] + 1} {t[1] + 1} {t[2] + 1}\n")
        if cnt % output_interval == 0 and (output_ply or output_obj):
            cnt_ply += 1
        cnt += 1
    ps._engine.check_status()
    dt = time.perf_counter() - t0
    if not args.quiet:
        print(f"{scene_name}: {ps.particle_max_num} particles, {cnt * substeps} steps in {dt:.3f} s "
              f"({cnt * substeps / dt:.1f} steps/s incl. exports)")
