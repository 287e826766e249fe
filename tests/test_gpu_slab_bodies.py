"""Sharded WCSPH scenes with dynamic solids on the GPU: a world-1 sharded run of the full armadillo_bath_dynamic
against the plain engine, the cube-body scene of tools/check_slab_parity.py on one rank, and two GPUs over NCCL against
one (skipped with fewer than two GPUs).

The plain engine's reactions are float atomics, so it need not repeat itself bit for bit; the armadillo tolerances are
stated against the spread of two plain runs measured in the same test: sharded vs plain <= max(1e-3 d, 2 x plain vs
plain) for positions and body centres of mass, and the same factor for R (floor 1e-3)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")


def _run(nproc, extra, port=29596):
    if nproc == 1:
        cmd = [sys.executable, SCRIPT, *extra]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), SCRIPT, *extra]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=dict(os.environ), cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


FLAG_FLUID, FLAG_DYNAMIC = 1, 2


def _plain(sc, steps, dev):
    from sph_taichi_b200 import ParticleSystem, SimConfig
    ps = ParticleSystem(SimConfig(sc), device=dev)
    s = ps.build_solver()
    s.initialize()
    s.step(steps)
    return ps


def _as_gathered(ps):
    """A plain engine's state in the layout of slab.gather_owned, for slab.compare_with_single."""
    import torch
    ps._pull()
    n = int(ps.particle_num[None])
    t = ps._t
    flags = (t["material"][:n] == 1).int() * FLAG_FLUID | (t["is_dynamic"][:n] != 0).int() * FLAG_DYNAMIC
    return (t["x"][:n].clone(), t["v"][:n].clone(), t["x_0"][:n].clone(), t["object_id"][:n].clone(),
            t["m_V"][:n].clone(), flags.to(torch.int32))


def _bodies_of(ps):
    out = {}
    for oid, b in ps._body_index.items():
        R, cm = ps._engine.rigid_state(b)
        out[oid] = (cm, R)
    return out


# The three armadillos start 0.35 m above the surface at -5 m/s and enter the fluid before step 200 (asserted below
# from the plain engine: each body's mean vertical velocity has left free fall by then).
ARMADILLO_STEPS = 200


def test_armadillo_bath_dynamic_single_rank_vs_plain_engine():
    """World 1, the whole armadillo_bath_dynamic (1.74 M particles, three shape-matched bodies) for 200 WCSPH steps,
    sharded against the plain engine, with the plain engine's own run-to-run spread as the yardstick."""
    import torch
    from sph_taichi_b200 import scene, slab
    dev = torch.device("cuda:0")
    sc = scene.NAMED_SCENES["armadillo_bath_dynamic"]()
    d = 2.0 * sc["Configuration"]["particleRadius"]
    sim, _ = slab.build_sharded(sc, 0, 1, dev, dynamic_solids=True)
    sim.step(ARMADILLO_STEPS)
    sim.info()  # raises on a status flag
    gathered = slab.gather_owned(sim)
    sharded_bodies = {oid: sim.body_state(b) for b, (oid, *_r) in enumerate(sim.bodies)}
    sim.eng.close()
    del sim
    ps1 = _plain(sc, ARMADILLO_STEPS, dev)
    cmp_s = slab.compare_with_single(gathered, ps1, d, bodies=sharded_bodies)
    del gathered
    ps2 = _plain(sc, ARMADILLO_STEPS, dev)
    cmp_p = slab.compare_with_single(_as_gathered(ps2), ps1, d, bodies=_bodies_of(ps2))
    del ps2
    g_y = float(sc["Configuration"]["gravitation"][1])
    t = ARMADILLO_STEPS * float(sc["Configuration"]["timeStepSize"])
    V, OID = _as_gathered(ps1)[1], _as_gathered(ps1)[3]
    for body in sc["RigidBodies"]:
        free = float(body["velocity"][1]) + g_y * t
        vy = float(V[OID == body["objectId"]][:, 1].double().mean())
        assert abs(vy - free) > 0.01 * abs(free), (body["objectId"], vy, free)
    msg = f"sharded vs plain {cmp_s}; plain vs plain {cmp_p}"
    assert cmp_s["same_particle_set"] and cmp_p["same_particle_set"], msg
    assert cmp_s["max_dx_over_d"] <= max(1e-3, 2 * cmp_p["max_dx_over_d"]), msg
    bp = {b["object_id"]: b for b in cmp_p["bodies"]}
    assert len(cmp_s["bodies"]) == 3, msg
    for b in cmp_s["bodies"]:
        p = bp[b["object_id"]]
        assert b["dcm_over_d"] <= max(1e-3, 2 * p["dcm_over_d"]), msg
        assert b["max_dR"] <= max(1e-3, 2 * p["max_dR"]), msg


def test_cube_body_scene_single_rank():
    """World 1, the cube body across the would-be cut and the dynamic block on the fluid surface, 20 steps."""
    out = _run(1, ["--dynamic-body", "--dynamic-block", "--counts", "24", "8", "8", "--steps", "20", "--vx", "3"])
    assert out["same_particle_set"] and out["max_dv"] < 1e-2 and out["reactions_acted"], out
    assert out["max_dx_over_d_fluid"] < 1e-3 and out["max_dx_over_d"] < 1e-3, out
    assert all(b["dcm_over_d"] < 1e-3 and b["max_dR"] < 1e-3 for b in out["bodies"]), out
    assert out["ok"], out


def test_cube_body_scene_two_gpus():
    """Two GPUs over NCCL against one engine: the cut runs through the body, cm and R are bit-identical on both
    ranks after every step."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    out = _run(2, ["--dynamic-body", "--dynamic-block", "--counts", "48", "12", "12", "--steps", "40", "--vx", "3"])
    assert out["same_particle_set"] and out["reactions_acted"] and out["bodies_bit_identical_across_ranks"], out
    lo, hi = out["body_layers"]
    assert lo < out["slabs_first"][0][1] < hi, out
    assert out["ok"], out
