"""The sharded engine's shape-matching solve against the plain engine's, bit for bit.

Bodies falling freely, clear of the fluid, move by the same arithmetic in both engines; only where the solve reads
their particles differs (k_rigid: the particle arrays, k_shard_body_solve: the all-gathered records).  So on a world-1
sharded context every body's cm and R and every body particle's position must equal the plain engine's after every
step; a moment reduction summed in any other order fails this (DESIGN.md section 4).  The two-cube scene also runs on
the host-emulated build of the same sources (tests/emu/)."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE = os.path.join(ROOT, "tests", "golden", "cube.obj")


def _device():
    import torch
    return torch.device("cpu") if os.environ.get("SPH_EMU_LIB") else torch.device("cuda:0")


def _cube(oid, lo, side, density):
    return {"objectId": oid, "geometryFile": CUBE, "translation": lo, "rotationAxis": [0, 1, 0], "rotationAngle": 0,
            "scale": [side] * 3, "velocity": [0.0, 0.0, 0.0], "density": density, "color": [255, 255, 255],
            "isDynamic": True}


def two_cubes_scene():
    """A 12 x 6 x 6 dam break (d = 0.02, surface at y = 0.18) and two cubes 0.1 above it: one of 11 d (more particles
    than the solve's 1024 threads, so threads sum more than one particle) over the fluid, one of 4.5 d beside it (the
    second body takes the first body's wall clamp before its solve)."""
    from sph_taichi_b200 import scene
    d = 0.02
    sc = scene.dam_break_box([12, 6, 6], domain_end=[0.9, 0.8, 0.45], start=[0.06] * 3)
    sc["RigidBodies"] = [_cube(1, [0.07, 0.28, 0.08], 11 * d, 800.0), _cube(2, [0.50, 0.28, 0.10], 4.5 * d, 600.0)]
    return sc


def _body_rows(x, x0, oid, ids):
    """Positions and x_0 of the particles of the objects ``ids``, ordered by (object_id, x_0)."""
    keep = np.isin(oid, ids)
    x, x0, oid = x[keep], x0[keep], oid[keep]
    order = np.lexsort((x0[:, 2], x0[:, 1], x0[:, 0], oid))
    return x[order], x0[order]


def run_in_lockstep(sc, steps):
    """Step a world-1 sharded context and the plain engine in lockstep, asserting bit-identical bodies after every
    step.  Returns the plain engine's largest |mean v_y - free fall| of a body after the last step."""
    from sph_taichi_b200 import ParticleSystem, SimConfig, slab
    dev = _device()
    sim, _ = slab.build_sharded(sc, 0, 1, dev, dynamic_solids=True)
    ps = ParticleSystem(SimConfig(sc), device=dev)
    solver = ps.build_solver()
    solver.initialize()
    ids = [oid for oid, *_rest in sim.bodies]
    assert sorted(ids) == sorted(b["objectId"] for b in sc["RigidBodies"]), ids
    moved = False
    for step in range(1, steps + 1):
        sim.step(1)
        solver.step(1)
        for b, oid in enumerate(ids):
            cm_s, R_s = sim.body_state(b)
            R_p, cm_p = ps._engine.rigid_state(ps._body_index[oid])
            assert np.array_equal(cm_s, cm_p), (step, oid, cm_s, cm_p)
            assert np.array_equal(R_s, R_p), (step, oid, R_s, R_p)
        x, _v, x0, oid = (t.cpu().numpy() for t in sim.owned_tensors()[:4])
        xs, x0s = _body_rows(x, x0, oid, ids)
        ps._pull()
        n = int(ps.particle_num[None])
        t = ps._t
        xp, x0p = _body_rows(t["x"][:n].cpu().numpy(), t["x_0"][:n].cpu().numpy(), t["object_id"][:n].cpu().numpy(),
                             ids)
        assert xs.shape[0] > 0 and np.array_equal(x0s, x0p), step
        assert np.array_equal(xs, xp), (step, float(np.abs(xs - xp).max()))
        moved = moved or not np.array_equal(xs, x0s)
    assert moved  # the bodies fell: positions left x_0
    sim.info()  # raises on a status flag
    g_y, dt = float(sc["Configuration"]["gravitation"][1]), float(sc["Configuration"]["timeStepSize"])
    oid_p, v_p = t["object_id"][:n].cpu().numpy(), t["v"][:n].cpu().numpy()
    dev_free = 0.0
    for body in sc["RigidBodies"]:
        free = float(body["velocity"][1]) + g_y * steps * dt
        dev_free = max(dev_free, abs(float(v_p[oid_p == body["objectId"]][:, 1].astype(np.float64).mean()) - free))
    return dev_free


@pytest.mark.gpu
def test_two_cubes_free_fall_sharded_vs_plain():
    """40 steps of the two cubes (8 on the much slower emulated build): still in free fall at the end (no fluid
    reached them)."""
    assert run_in_lockstep(two_cubes_scene(), 8 if os.environ.get("SPH_EMU_LIB") else 40) < 1e-4


@pytest.mark.gpu
def test_armadillo_bath_dynamic_before_the_impact():
    """The full armadillo_bath_dynamic (1.74 M particles, three shape-matched bodies): the first 60 steps, while the
    armadillos fall toward the surface at -5 m/s."""
    from sph_taichi_b200 import scene
    assert run_in_lockstep(scene.NAMED_SCENES["armadillo_bath_dynamic"](), 60) < 1e-3


def test_two_cubes_on_the_emulated_build():
    """test_two_cubes_free_fall_sharded_vs_plain against the host-emulated build of the same sources."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    env = dict(os.environ, SPH_EMU_LIB=build_emu.build(), PYTHONPATH=ROOT)
    env.pop("SPH_B200_LIB", None)
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "-k", "two_cubes_free_fall",
           os.path.abspath(__file__)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env, cwd=ROOT)
    tail = res.stdout[-3000:] + res.stderr[-3000:]
    assert res.returncode == 0 and "1 passed" in res.stdout, tail
