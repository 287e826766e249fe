"""Scene dictionaries (the reference's JSON schema) and initial-condition assembly.

* ``dragon_bath`` / ``armadillo_bath_dynamic`` / ``high_fluid_wcsph`` reproduce the
  parameter sets of the reference's WCSPH scenes (``data/scenes/*.json``), with one
  extra optional key per rigid body, ``voxelizedPointsFile``: a committed lattice
  fixture (``sph_taichi_b200/data/rigid/*.npz``, produced by
  ``tools/make_rigid_fixtures.py`` with ``voxelizer.py``) used when the mesh file
  named by ``geometryFile`` is not on disk (the reference's ``data/models`` are not
  redistributed here and do not exist on the GPU box).
* ``dam_break_box`` builds the synthetic BASELINE configs (8 K cube, 4 M and 16 M
  boxes; SURVEY.md section 8d).
* ``assemble_particles`` restates the particle ordering and per-particle values of
  the reference constructor (``particle_system.py:54-83,151-211,450-495``): fluid
  blocks, then rigid blocks, then rigid bodies.
"""
from __future__ import annotations

import json
import os
from functools import reduce

import numpy as np

from . import voxelizer

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))


def _base_configuration(domain_end, **over):
    cfg = {
        "domainStart": [0.0, 0.0, 0.0],
        "domainEnd": [float(v) for v in domain_end],
        "particleRadius": 0.01,
        "numberOfStepsPerRenderUpdate": 1,
        "density0": 1000,
        "simulationMethod": 0,
        "gravitation": [0.0, -9.81, 0.0],
        "timeStepSize": 0.0004,
        "stiffness": 50000,
        "exponent": 7,
        "boundaryHandlingMethod": 0,
        "exportFrame": False,
        "exportPly": False,
        "exportObj": False,
    }
    cfg.update(over)
    return cfg


def _fluid_block(start, end, translation=(0.0, 0.0, 0.0), velocity=(0.0, 0.0, 0.0), object_id=0):
    return {
        "objectId": object_id,
        "start": [float(v) for v in start],
        "end": [float(v) for v in end],
        "translation": [float(v) for v in translation],
        "scale": [1, 1, 1],
        "velocity": [float(v) for v in velocity],
        "density": 1000.0,
        "color": [50, 100, 200],
    }


def _rigid_body(object_id, geometry, fixture, translation, angle, scale, velocity, density, color, dynamic):
    return {
        "objectId": object_id,
        "geometryFile": geometry,
        "voxelizedPointsFile": fixture,
        "translation": [float(v) for v in translation],
        "rotationAxis": [0, 1, 0],
        "rotationAngle": angle,
        "scale": list(scale),
        "velocity": [float(v) for v in velocity],
        "density": float(density),
        "color": list(color),
        "isDynamic": bool(dynamic),
    }


def dragon_bath(with_rigid=True):
    """423 500 fluid particles falling at 1 m/s around a static dragon (BASELINE cfg 2)."""
    scene = {
        "Configuration": _base_configuration([5.0, 3.0, 2.0]),
        "FluidBlocks": [_fluid_block([0.1, 0.1, 0.5], [1.2, 2.9, 1.6], translation=[0.2, 0.0, 0.2],
                                     velocity=[0.0, -1.0, 0.0])],
    }
    if with_rigid:
        scene["RigidBodies"] = [
            _rigid_body(1, "./data/models/Dragon_50k.obj", "../rigid/dragon_bath_1.npz", [3.5, 0.05, 1.0], 0,
                        [1, 1, 1], [0.0, 0.0, 0.0], 1000.0, [255, 255, 255], False)
        ]
    return scene


def armadillo_bath_dynamic():
    """1 723 968 fluid particles + three dynamic armadillos (BASELINE cfg 3)."""
    bodies = []
    for oid, tx, rho, col in ((1, 4.0, 7874.0, [255, 255, 255]), (2, 2.5, 1700.0, [255, 100, 50]),
                              (3, 1.0, 300.0, [100, 100, 50])):
        bodies.append(_rigid_body(oid, "./data/models/armadillo_small.obj", f"../rigid/armadillo_bath_{oid}.npz",
                                  [tx, 2.0, 1.2], 180, [0.25, 0.25, 0.25], [0.0, -5.0, 0.0], rho, col, True))
    return {
        "Configuration": _base_configuration([5.0, 3.0, 2.0]),
        "RigidBodies": bodies,
        "FluidBlocks": [_fluid_block([0.04, 0.04, 0.04], [4.96, 1.50, 1.96])],
    }


def high_fluid_wcsph():
    return {
        "Configuration": _base_configuration([2.0, 6.0, 2.0]),
        "FluidBlocks": [_fluid_block([0.0, 0.0, 0.0], [0.6, 5.4, 0.6], translation=[0.1, 0.1, 0.1])],
    }


def dam_break_box(counts, domain_end=None, start=None, radius=0.01, **over):
    """Synthetic lattice dam break with ``counts`` particles per axis.

    The block end is placed half a spacing short of ``start + counts * d`` so that the
    ``np.arange`` rule of the reference (``particle_system.py:450-456``) yields exactly
    ``counts`` regardless of floating-point step accumulation; ``assemble_particles``
    re-checks the count.
    """
    d = 2.0 * radius
    counts = [int(c) for c in counts]
    if start is None:
        start = [4.0 * radius] * 3
    end = [s + (c - 0.5) * d for s, c in zip(start, counts)]
    if domain_end is None:
        domain_end = [2.0 * s + c * d for s, c in zip(start, counts)]
    scene = {
        "Configuration": _base_configuration(domain_end, particleRadius=radius, **over),
        "FluidBlocks": [_fluid_block(start, end)],
    }
    return scene


def cube_8k():
    """BASELINE cfg 1: 20^3 lattice in a unit box (SURVEY.md section 8d)."""
    return dam_break_box([20, 20, 20], domain_end=[1.0, 1.0, 1.0], start=[0.1, 0.1, 0.1])


def box_4m():
    """BASELINE cfg 4: 200 x 100 x 200 = 4.0 M particles, domain 8.08 x 3.0 x 4.08."""
    return dam_break_box([200, 100, 200], domain_end=[8.08, 3.0, 4.08], start=[0.04, 0.04, 0.04])


def box_16m():
    """BASELINE cfg 5: 400 x 100 x 400 = 16.0 M particles, domain 16.08 x 3.0 x 8.08."""
    return dam_break_box([400, 100, 400], domain_end=[16.08, 3.0, 8.08], start=[0.04, 0.04, 0.04])


def _as_dfsph(sc, dt=0.004):
    sc["Configuration"]["simulationMethod"] = 4
    sc["Configuration"]["timeStepSize"] = dt
    return sc


def _as_iisph(sc, dt=0.001):
    sc["Configuration"]["simulationMethod"] = 3
    sc["Configuration"]["timeStepSize"] = dt
    return sc


def _as_pcisph(sc, dt=0.001):
    sc["Configuration"]["simulationMethod"] = 1
    sc["Configuration"]["timeStepSize"] = dt
    return sc


def dragon_bath_pcisph():
    """dragon_bath's geometry with the PCISPH solver (simulationMethod 1), dt = 1e-3 (DESIGN.md section 11)."""
    return _as_pcisph(dragon_bath())


def dragon_bath_iisph():
    """dragon_bath's geometry with the IISPH solver (simulationMethod 3), dt = 1e-3 (DESIGN.md section 10)."""
    return _as_iisph(dragon_bath())


def dragon_bath_dfsph():
    """The reference's dragon_bath_dfsph.json: same geometry, DFSPH, dt = 4e-3."""
    return _as_dfsph(dragon_bath())


def dragon_bath_dynamic_dfsph():
    """The reference's dragon_bath_dynamic_dfsph.json: the dragon is a dynamic (shape-matched) body."""
    sc = dragon_bath_dfsph()
    for body in sc["RigidBodies"]:
        body["isDynamic"] = True
    return sc


def high_fluid_dfsph():
    return _as_dfsph(high_fluid_wcsph())


def armadillo_bath_dynamic_dfsph():
    return _as_dfsph(armadillo_bath_dynamic())


def armadillo_bath_dynamic_iisph():
    """armadillo_bath_dynamic's geometry (three shape-matched armadillos) with the IISPH solver, dt = 1e-3: the
    full-size scene of sharded IISPH with dynamic solids."""
    return _as_iisph(armadillo_bath_dynamic())


def box_4m_dfsph():
    """box_4m with the DFSPH solver (dt = 4e-3): the sharded DFSPH workload of bench.py --gpus N."""
    return _as_dfsph(box_4m())


NAMED_SCENES = {
    "dragon_bath": dragon_bath,
    "armadillo_bath_dynamic": armadillo_bath_dynamic,
    "high_fluid_wcsph": high_fluid_wcsph,
    "dragon_bath_dfsph": dragon_bath_dfsph,
    "dragon_bath_iisph": dragon_bath_iisph,
    "dragon_bath_pcisph": dragon_bath_pcisph,
    "dragon_bath_dynamic_dfsph": dragon_bath_dynamic_dfsph,
    "high_fluid_dfsph": high_fluid_dfsph,
    "armadillo_bath_dynamic_dfsph": armadillo_bath_dynamic_dfsph,
    "armadillo_bath_dynamic_iisph": armadillo_bath_dynamic_iisph,
    "cube_8k": cube_8k,
    "box_4m": box_4m,
    "box_16m": box_16m,
    "box_4m_dfsph": box_4m_dfsph,
}


def write_scene_files(out_dir=None):
    """Materialise the named scenes as JSON files (``python -m sph_taichi_b200.scene [out_dir]``).

    The files are generated, not committed: they necessarily carry the reference's parameter values."""
    out_dir = out_dir or os.path.join(_PKG_DIR, "data", "scenes")
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in NAMED_SCENES.items():
        with open(os.path.join(out_dir, name + ".json"), "w") as fh:
            json.dump(fn(), fh, indent=2)
            fh.write("\n")


# ---------------------------------------------------------------------------------
# initial conditions
# ---------------------------------------------------------------------------------

def cube_axis_samples(lower, size, diameter):
    """Per-axis lattice coordinates: ``np.arange(lo, lo + size, d)`` (particle_system.py:469-473)."""
    return [np.arange(lower[i], lower[i] + size[i], diameter) for i in range(len(lower))]


def cube_particle_count(start, end, diameter):
    """``compute_cube_particle_num`` (particle_system.py:450-456)."""
    return reduce(lambda a, b: a * b, [len(np.arange(start[i], end[i], diameter)) for i in range(len(start))])


def cube_positions(lower, size, diameter):
    """float32 lattice positions in meshgrid 'ij' order, x slowest (particle_system.py:478-483)."""
    axes = cube_axis_samples(lower, size, diameter)
    grid = np.array(np.meshgrid(*axes, sparse=False, indexing="ij"), dtype=np.float32)
    return np.ascontiguousarray(grid.reshape(len(axes), -1).T)


def rigid_body_lattice(body, diameter, scene_dir):
    """Lattice indices of a ``RigidBodies`` entry: mesh if present, else committed fixture."""
    geom = body.get("geometryFile")
    cands = []
    if geom:
        cands += [geom, os.path.join(scene_dir, geom), os.path.join(scene_dir, "..", "..", geom)]
    for path in cands:
        if os.path.isfile(path):
            idx, verts, faces, weights = voxelizer.voxelize_rigid_body(
                path, body["scale"], body["rotationAngle"], body["rotationAxis"], body["translation"], diameter)
            body["_vertexWeights"] = weights  # trimesh's vertex multiplicity (rest centre of mass, voxelizer.load_obj)
            return idx, verts, faces
    fix = body.get("voxelizedPointsFile")
    if fix:
        for path in (fix, os.path.join(scene_dir, fix), os.path.join(_PKG_DIR, "data", "rigid", os.path.basename(fix))):
            path = os.path.normpath(path)
            if os.path.isfile(path):
                with np.load(path) as z:
                    if abs(float(z["pitch"]) - diameter) > 1e-12:
                        raise ValueError(f"{path}: fixture pitch {float(z['pitch'])} != particle diameter {diameter}")
                    return z["lattice"].astype(np.int64), None, None
    raise FileNotFoundError(
        f"rigid body {body.get('objectId')}: neither geometryFile {geom!r} nor voxelizedPointsFile {fix!r} found")


def assemble_particles(cfg, dim, diameter, verbose=False):
    """Build all initial per-particle arrays in the reference's order.

    Returns ``(arrays, object_collection, object_id_rigid_body, counts)`` where
    ``arrays`` holds float32/int32 numpy arrays: object_id, x, v, density, pressure,
    material, is_dynamic, color.
    """
    parts = []
    object_collection = {}
    rigid_ids = set()

    def block(spec, material, is_dynamic):
        offset = np.array(spec["translation"])
        start = np.array(spec["start"]) + offset
        end = np.array(spec["end"]) + offset
        scale = np.array(spec["scale"])
        pos = cube_positions(start, (end - start) * scale, diameter)
        declared = cube_particle_count(spec["start"], spec["end"], diameter)
        if declared != pos.shape[0]:
            # the reference sizes its fields from the untranslated count and fills from the
            # translated one (particle_system.py:57 vs :160); a mismatch overruns its fields.
            raise ValueError(f"object {spec['objectId']}: lattice count {pos.shape[0]} != declared {declared}")
        n = pos.shape[0]
        spec["particleNum"] = n
        object_collection[spec["objectId"]] = spec
        vel = spec.get("velocity")
        v = np.zeros_like(pos) if vel is None else np.tile(np.asarray(vel, dtype=np.float32), (n, 1))
        dens = spec.get("density")
        parts.append(dict(
            object_id=np.full(n, spec["objectId"], np.int32), x=pos, v=v,
            density=np.full(n, 1000.0 if dens is None else dens, np.float32),
            pressure=np.zeros(n, np.float32), material=np.full(n, material, np.int32),
            is_dynamic=np.full(n, int(is_dynamic), np.int32),
            color=np.tile(np.asarray(spec["color"], dtype=np.int32), (n, 1))))
        if verbose:
            print("particle num ", n)
        return n

    n_fluid = sum(block(f, 1, 1) for f in cfg.get_fluid_blocks())
    n_rigid = sum(block(r, 0, r["isDynamic"]) for r in cfg.get_rigid_blocks())
    for body in cfg.get_rigid_bodies():
        lattice, verts, faces = rigid_body_lattice(body, diameter, cfg.scene_dir)
        pts64 = lattice.astype(np.float64) * diameter
        n = pts64.shape[0]
        body["particleNum"] = n
        body["voxelizedPoints"] = pts64
        if verts is not None:
            body["restPosition"] = verts
            body["restCenterOfMass"] = voxelizer.vertex_mean(verts, body.get("_vertexWeights"))
            body["meshFaces"] = faces
        object_collection[body["objectId"]] = body
        rigid_ids.add(body["objectId"])
        dyn = int(bool(body["isDynamic"]))
        vel = np.asarray(body["velocity"], np.float32) if dyn else np.zeros(dim, np.float32)
        parts.append(dict(
            object_id=np.full(n, body["objectId"], np.int32), x=pts64.astype(np.float32),
            v=np.tile(vel, (n, 1)), density=np.full(n, body["density"], np.float32),
            pressure=np.zeros(n, np.float32), material=np.zeros(n, np.int32),
            is_dynamic=np.full(n, dyn, np.int32),
            color=np.tile(np.asarray(body["color"], dtype=np.int32), (n, 1))))
        n_rigid += n
        if verbose:
            print(f"rigid body {body['objectId']} num: {n}")

    keys = ("object_id", "x", "v", "density", "pressure", "material", "is_dynamic", "color")
    if parts:
        arrays = {k: np.ascontiguousarray(np.concatenate([p[k] for p in parts], axis=0)) for k in keys}
    else:
        arrays = {k: np.zeros((0, 3) if k in ("x", "v", "color") else (0,), np.float32) for k in keys}
    counts = dict(fluid=n_fluid, solid=n_rigid, total=n_fluid + n_rigid)
    return arrays, object_collection, rigid_ids, counts


if __name__ == "__main__":
    import sys
    write_scene_files(sys.argv[1] if len(sys.argv) > 1 else None)
    print("wrote", ", ".join(sorted(NAMED_SCENES)))
