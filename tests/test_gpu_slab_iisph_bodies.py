"""Sharded IISPH with dynamic solids (sph_shard_configure_iisph_bodies, build_sharded(iisph_bodies=True)) on the GPU:
world-1 sharded runs against the plain IISPH engine on the cube-body scene of tools/check_slab_parity.py, the reaction
gather against the plain engine's scatter after one step from the same state, armadillo_bath_dynamic_iisph at full
size, two GPUs over NCCL against one (skipped with fewer than two GPUs), and the refusals on a CUDA context.

All but the full-size test also run against the host-emulated library (SPH_EMU_LIB)."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")
sys.path.insert(0, os.path.join(ROOT, "tools"))
D = 0.02
FLAG_FLUID, FLAG_DYNAMIC = 1, 2


def _dev():
    import torch
    return torch.device("cpu") if os.environ.get("SPH_EMU_LIB") else torch.device("cuda:0")


def _run(nproc, extra, timeout=1500):
    args = [SCRIPT, "--iisph", "--dynamic-body", "--dynamic-block", *extra]
    if nproc == 1:
        cmd = [sys.executable, *args]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", "29587", *args]
    env = dict(os.environ, SPH_SHARD_GRAPH="0")  # SPH_EMU_LIB, if set, routes the tool to the emulated library
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check(out):
    assert out["same_particle_set"] and out["dynamic_solids"] > 0 and out["n_bodies"] == 1, out
    assert out["iterations_sharded"] == out["iterations_single"], out  # the same sweeps in every step
    assert out["max_dx_over_d_fluid"] < 1e-3 and out["max_dx_over_d"] < 1e-3 and out["max_dv"] < 1e-2, out
    assert all(b["dcm_over_d"] < 1e-3 and b["max_dR"] < 1e-3 for b in out["bodies"]), out
    assert out["reactions_acted"] and out["status"] == [0] * out["world"], out  # no flag, the velocity flag included
    assert out["ok"], out


def test_cube_body_scene_single_rank_equals_plain_engine():
    """World 1, fluid at +3 m/s under the shape-matched cube and the dynamic block, 40 steps: the plain engine's sweep
    count in every step, fluid and solids within 1e-3 d, cm and R within 1e-3, and a status word of 0 -- a body does
    not trip the velocity flag that k_iisph_advect now also raises for dynamic solids."""
    _check(_run(1, ["--counts", "24", "8", "8", "--steps", "40", "--vx", "3"]))


def _pressed_scene():
    """The cube and the block lowered to 0.85 spacings above the fluid's top layer: the fluid under them is above rho0
    in the very first step, so its pressures -- and the reactions -- are non-zero after one step from the start."""
    from check_slab_parity import add_dynamic_solids
    from sph_taichi_b200 import scene
    c = [16, 8, 8]
    sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * D + 0.2, c[1] * D + 0.4, c[2] * D + 0.12], start=[0.06] * 3)
    sc = add_dynamic_solids(sc, c, D, 1, True, True)
    sc["RigidBodies"][0]["translation"][1] -= 0.4 * D
    for k in ("start", "end"):
        sc["RigidBlocks"][0][k][1] -= 0.15 * D
    return scene._as_iisph(sc)


def test_reaction_gather_equals_the_plain_engines_scatter():
    """One step from the same state: acc of every dynamic solid = g + reactions, gathered by k_iisph_shard_reactions in
    the sharded world-1 context and scattered with float atomics by k_iisph_pressure_accel<true> in the plain engine.
    Only the summation order differs: equal within 1e-4 of the largest reaction, and not all g."""
    import numpy as np
    import torch
    from sph_taichi_b200 import ParticleSystem, SimConfig, slab
    dev = _dev()
    sc = _pressed_scene()
    g = np.array(sc["Configuration"]["gravitation"], np.float32)
    ps = ParticleSystem(SimConfig(sc), device=dev)
    solver = ps.build_solver()
    solver.initialize()
    solver.step(1)
    ps._pull()
    n = int(ps.particle_num[None])
    t = ps._t
    dyn = (t["material"][:n] != 1) & (t["is_dynamic"][:n] != 0)
    a1, x01, oid1 = (t[k][:n][dyn].cpu().numpy() for k in ("acceleration", "x_0", "object_id"))
    sim, _ = slab.build_sharded(_pressed_scene(), 0, 1, dev, iisph_bodies=True)
    sim.step(1)
    sim.synchronize()
    info = sim.info()
    assert info["status"] == 0, info
    off = (C.c_uint64 * 5)()
    e = sim.eng
    e._check(e.lib.sph_state_offsets(e.ctx, off), "sph_state_offsets")
    b0 = e._ws_ptr - e.workspace.data_ptr() + int(off[4])
    acc = e.workspace[b0:b0 + sim.n_cap * 16].view(torch.float32).view(sim.n_cap, 4)
    rec = sim.record_views()
    own = slice(info["own_begin"], info["own_end"])
    flags = rec[3][own, 2].contiguous().view(torch.int32)
    m = (flags & (FLAG_FLUID | FLAG_DYNAMIC)) == FLAG_DYNAMIC
    a2, x02 = acc[own][m].cpu().numpy(), rec[2][own, :3][m].cpu().numpy()
    oid2 = rec[2][own, 3].contiguous().view(torch.int32)[m].cpu().numpy()
    assert a2.shape[0] == a1.shape[0] > 0, (a1.shape, a2.shape)
    k1, k2 = (np.lexsort((x[:, 2], x[:, 1], x[:, 0], o)) for x, o in ((x01, oid1), (x02, oid2)))
    assert np.array_equal(x01[k1], x02[k2])
    assert np.all(a2[:, 3] == 0.0)  # acc.w of a solid stays 0 (k_iisph_pressure_update relies on it)
    r1, r2 = a1[k1] - g, a2[k2][:, :3] - g  # the reactions
    largest = float(np.abs(r1).max())
    assert largest > 1e-2 * float(np.abs(g).max()), largest  # not all g
    assert float(np.abs(r1 - r2).max()) <= 1e-4 * largest, (float(np.abs(r1 - r2).max()), largest)
    e.close()


def _plain_run(sc, steps, dev):
    """The plain engine for `steps` steps, one per call: (ParticleSystem, sweep count of every step)."""
    from sph_taichi_b200 import ParticleSystem, SimConfig
    ps = ParticleSystem(SimConfig(sc), device=dev)
    s = ps.build_solver()
    s.initialize()
    counts = []
    for _ in range(steps):
        s.step(1)
        counts.append(int(s.last_iterations))
    return ps, counts


# The three armadillos fall at -5 m/s and come within the support radius of the surface after about 50 steps of
# dt = 1e-3.  From there the scene is violent in IISPH at this time step, in the plain engine too: single body particles
# reach tens of m/s within a few steps (the shape matching moves positions, not velocities), the plain engine's
# pressure loop hits its cap at step 74 and it leaves the grid at step 76 (H100).  The sharded engine stops earlier, at
# step 58, on its velocity bound (a body particle above h / dt = 40 m/s in x).  The comparison therefore runs to step
# 55: the reactions already act (asserted below from the plain engine) and neither engine has raised a flag.
ARMADILLO_STEPS = 55


@pytest.mark.skipif(bool(os.environ.get("SPH_EMU_LIB")), reason="full size: GPU only")
def test_full_size_armadillo_bath_dynamic_iisph():
    """armadillo_bath_dynamic_iisph (1.74 M particles, three shape-matched bodies), world 1, 55 steps (chosen above),
    sharded against the plain engine.  The plain engine's reactions are float atomics, so two runs of it need not agree:
    its own spread is measured here and is the yardstick.  Sweep counts: equal step by step up to the first step at
    which the two plain runs differ (all 55 if they never do).  Positions, body centres of mass and R: within
    max(1e-3 d, 2 x plain vs plain), floor 1e-3 for R."""
    import torch
    from tests.test_gpu_slab_bodies import _as_gathered, _bodies_of
    from sph_taichi_b200 import scene, slab
    dev = torch.device("cuda:0")
    sc = scene.NAMED_SCENES["armadillo_bath_dynamic_iisph"]()
    d = 2.0 * sc["Configuration"]["particleRadius"]
    sim, _ = slab.build_sharded(sc, 0, 1, dev, iisph_bodies=True)
    counts_s = []
    for _ in range(ARMADILLO_STEPS):
        sim.step(1)
        counts_s.append(sim.last_iterations)
    assert sim.info()["status"] == 0
    gathered = slab.gather_owned(sim)
    sharded_bodies = {oid: sim.body_state(b) for b, (oid, *_r) in enumerate(sim.bodies)}
    sim.eng.close()
    del sim
    ps1, counts_1 = _plain_run(sc, ARMADILLO_STEPS, dev)
    cmp_s = slab.compare_with_single(gathered, ps1, d, bodies=sharded_bodies)
    del gathered
    ps2, counts_2 = _plain_run(sc, ARMADILLO_STEPS, dev)
    cmp_p = slab.compare_with_single(_as_gathered(ps2), ps1, d, bodies=_bodies_of(ps2))
    del ps2
    g_y = float(sc["Configuration"]["gravitation"][1])
    t = ARMADILLO_STEPS * float(sc["Configuration"]["timeStepSize"])
    V, OID = _as_gathered(ps1)[1], _as_gathered(ps1)[3]
    left = {}
    for body in sc["RigidBodies"]:  # the largest departure of a body particle's velocity from free fall
        v = V[OID == body["objectId"]].double()
        v[:, 1] -= float(body["velocity"][1]) + g_y * t
        left[body["objectId"]] = float(v.abs().max())
    assert max(left.values()) > 1.0, left  # reactions acted (m/s)
    same = next((k for k in range(ARMADILLO_STEPS) if counts_1[k] != counts_2[k]), ARMADILLO_STEPS)
    msg = (f"departure from free fall {left}; sharded vs plain {cmp_s}; plain vs plain {cmp_p}; plain runs' sweep counts agree for {same} steps; "
           f"sweeps sharded {counts_s} plain {counts_1}")
    assert counts_s[:same] == counts_1[:same], msg
    assert cmp_s["same_particle_set"] and cmp_p["same_particle_set"], msg
    assert cmp_s["max_dx_over_d"] <= max(1e-3, 2 * cmp_p["max_dx_over_d"]), msg
    bp = {b["object_id"]: b for b in cmp_p["bodies"]}
    assert len(cmp_s["bodies"]) == 3, msg
    for b in cmp_s["bodies"]:
        p = bp[b["object_id"]]
        assert b["dcm_over_d"] <= max(1e-3, 2 * p["dcm_over_d"]), msg
        assert b["max_dR"] <= max(1e-3, 2 * p["max_dR"]), msg


def test_cube_body_scene_two_gpus():
    """Two GPUs over NCCL against one engine: the cut runs through the body, sweep counts, cm and R are bit-identical
    on both ranks after every step."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    out = _run(2, ["--counts", "24", "8", "8", "--steps", "40", "--vx", "3"])
    _check(out)
    assert out["bodies_bit_identical_across_ranks"] and out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    lo, hi = out["body_layers"]
    assert lo < out["slabs_first"][0][1] < hi, out


def test_refusals_on_a_body_context():
    """sph_shard_configure_iisph_bodies refuses WCSPH and DFSPH contexts and ghost_layers < 3; on the context it
    configured, the solid-id entry points, the other sharded steps and the single-GPU IISPH calls are refused, and the
    context steps on afterwards."""
    import numpy as np
    from check_slab_parity import add_dynamic_solids
    from sph_taichi_b200 import SimConfig, _lib, engine, scene, slab
    dev = _dev()
    c = [12, 6, 6]

    def dyn_scene():
        sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * D + 0.2, c[1] * D + 0.4, c[2] * D + 0.12], start=[0.06] * 3)
        return add_dynamic_solids(sc, c, D, 1, True, True)

    def packed(mode):
        cfg = SimConfig(dyn_scene())
        arrays, _, _, counts = scene.assemble_particles(cfg, 3, D)
        arrays["solid_id"] = slab.solid_ids(arrays)
        n, ns = counts["total"], counts["solid"]
        e = engine.Engine(slab.scene_params(cfg), n_max=4 * n, n_solid=ns, n_bodies=1, device=dev)
        if mode == "dfsph":
            e.set_dfsph(True)
        if mode == "iisph":
            e.set_iisph(True)
        e.pack(slab.field_tensors(arrays, n, float(np.float32(0.8 * D ** 3)), dev), n, ns, True)
        assert e.lib.sph_comm_set_transport(e.ctx, None, 0, 1) == 0
        body = (_lib.SphRigidBody * 1)()
        body[0].object_id, body[0].solid_begin, body[0].solid_end = slab.dynamic_bodies(cfg, arrays)[0]
        body[0].rest_cm = (C.c_float * 3)(0.3, 0.3, 0.15)
        return e, int(slab.scene_params(cfg).grid_num[0]), n, body

    def refused(e, rc, what):
        msg = e.lib.sph_last_error(e.ctx)
        assert rc != 0 and what in msg, (rc, msg)

    for mode in ("wcsph", "dfsph"):
        e, gx, n, body = packed(mode)
        refused(e, e.lib.sph_shard_configure_iisph_bodies(e.ctx, 0, gx, 3, n, 8, body, 1), b"sph_set_iisph(1) before it")
        e.close()
    e, gx, n, body = packed("iisph")
    st = e._stream()
    refused(e, e.lib.sph_shard_configure_iisph_bodies(e.ctx, 0, gx, 2, n, 8, body, 1), b"ghost_layers >= 3")
    refused(e, e.lib.sph_shard_configure_bodies(e.ctx, 0, gx, 3, n, 8, body, 1), b"sph_shard_configure_iisph_bodies")
    e.close()
    sim, _ = slab.build_sharded(scene._as_iisph(dyn_scene()), 0, 1, dev, iisph_bodies=True)
    e = sim.eng
    st = e._stream()
    sim.step(2)
    io = _lib.SphIisphStep(max_iterations=100, omega=0.5, eta=1e-3, n_fluid=c[0] * c[1] * c[2], first_batch=2)
    dio = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
    it, avg = C.c_int32(0), C.c_double(0.0)
    refused(e, e.lib.sph_set_rigid_bodies(e.ctx, body, 1), b"static solids only")
    refused(e, e.lib.sph_set_rigid_bodies(e.ctx, body, 0), b"fixed")
    refused(e, e.lib.sph_boundary_volume(e.ctx, 1, st), b"static solids only")
    refused(e, e.lib.sph_compute_rigid_rest_cm(e.ctx, 0, st), b"static solids only")
    refused(e, e.lib.sph_solve_constraints(e.ctx, 0, None, st), b"static solids only")
    refused(e, e.lib.sph_shard_step(e.ctx, 1, st), b"sph_shard_iisph_step")
    refused(e, e.lib.sph_shard_profile_step(e.ctx, (C.c_float * 6)(), st), b"sph_shard_iisph_step")
    refused(e, e.lib.sph_shard_dfsph_step(e.ctx, 1, C.byref(dio), st), b"sph_shard_iisph_step")
    refused(e, e.lib.sph_iisph_step(e.ctx, 1, C.byref(io), st), b"sph_shard_iisph_step")
    refused(e, e.lib.sph_iisph_op(e.ctx, 1, 0.0, None, st), b"sph_shard_iisph_step")
    refused(e, e.lib.sph_iisph_solve(e.ctx, 1, 0.5, 1e-3, 1, 1, C.byref(it), C.byref(avg), st), b"sph_shard_iisph_step")
    sim.step(2)  # still usable
    sim.synchronize()
    assert sim.info()["owned"] == sim.object_counts[0] + sim.object_counts[2] + sim.object_counts[3]
    status = C.c_uint32(1)
    assert e.lib.sph_read_status(e.ctx, C.byref(status), st) == 0 and status.value == 0, status.value
    R, cm = e.rigid_state(0)
    assert np.isfinite(cm).all() and abs(np.linalg.det(R) - 1.0) < 1e-4, (R, cm)
    e.close()
