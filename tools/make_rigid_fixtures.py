"""Generate the committed rigid-body lattice fixtures and scene JSON files.

Run in the authoring container (needs the reference's mesh assets, which are NOT
copied into this repo):

    python tools/make_rigid_fixtures.py <checkout of erizmr/SPH_Taichi>

For every ``RigidBodies`` entry of the bath scenes it runs ``voxelizer.py`` on the
reference mesh with the scene's transform and stores the filled lattice indices
(int16) plus the pitch in ``sph_taichi_b200/data/rigid/<scene>_<objectId>.npz``.
Points are ``lattice * pitch``.

It also writes what the tests compare against without the reference tree: the reference's
scene files, copied unchanged to ``tests/golden/reference_scenes/``, and, per body,
the vertex multiplicities ``load_obj`` finds in the mesh and the plain (unweighted)
vertex mean after the scene's transform, in ``tests/golden/reference_meshes.json``.
"""
import json
import os
import shutil
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sph_taichi_b200 import scene, voxelizer  # noqa: E402


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: python tools/make_rigid_fixtures.py <checkout of erizmr/SPH_Taichi>")
    ref = sys.argv[1]
    out = os.path.join(os.path.dirname(scene.__file__), "data", "rigid")
    os.makedirs(out, exist_ok=True)
    gold = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
    os.makedirs(os.path.join(gold, "reference_scenes"), exist_ok=True)
    scenes = os.path.join(ref, "data", "scenes")
    for f in sorted(os.listdir(scenes)):
        if f.endswith(".json"):
            shutil.copyfile(os.path.join(scenes, f), os.path.join(gold, "reference_scenes", f))
    meshes = {}
    for name in ("dragon_bath", "armadillo_bath_dynamic"):
        sc = scene.NAMED_SCENES[name]()
        pitch = 2.0 * sc["Configuration"]["particleRadius"]
        for body in sc["RigidBodies"]:
            mesh = os.path.join(ref, body["geometryFile"])
            idx, verts, _, weights = voxelizer.voxelize_rigid_body(
                mesh, body["scale"], body["rotationAngle"], body["rotationAxis"], body["translation"], pitch)
            assert np.abs(idx).max() < 32767
            dst = os.path.join(out, os.path.basename(body["voxelizedPointsFile"]))
            np.savez_compressed(dst, lattice=idx.astype(np.int16), pitch=np.float64(pitch),
                                rest_center_of_mass=voxelizer.vertex_mean(verts, weights))
            print(f"{name} body {body['objectId']}: {idx.shape[0]} voxels -> {dst}")
            v, _, w = voxelizer.load_obj(mesh, with_multiplicity=True)
            moved = voxelizer.transform_rigid_mesh(v, body["scale"], body["rotationAngle"], body["rotationAxis"],
                                                   body["translation"])
            vals, cnts = np.unique(w, return_counts=True)
            meshes[os.path.basename(dst)] = {
                "geometryFile": body["geometryFile"], "vertices": int(len(v)),
                "vertex_multiplicity_histogram": {str(int(a)): int(c) for a, c in zip(vals, cnts)},
                "plain_vertex_mean_after_transform": [float(t) for t in moved.mean(0)]}
    with open(os.path.join(gold, "reference_meshes.json"), "w") as fh:
        json.dump(meshes, fh, indent=1)


if __name__ == "__main__":
    main()
