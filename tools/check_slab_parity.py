"""Sharded engine vs single-GPU engine on the same scene (run under torchrun, 1 rank per GPU).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29533 tools/check_slab_parity.py --counts 64 24 24 --steps 60

Rank 0 also runs the plain single-GPU engine and compares every particle (matched by object_id and x_0).
Prints one JSON line and exits non-zero on mismatch.

--static-block puts a static rigid block under the fluid, across every cut; the tool then also checks that every
static solid is still exactly at x_0 with the single engine's start-up boundary volume m_V.

--dfsph runs the scene with the DFSPH solver (dt = 4e-3) and also compares the Jacobi iteration counts of every step
with the single engine's, checks that every rank reported bit-identical counts and average errors in every step, and
that after the last step's ghost alignment each ghost record holds the x_0 of the neighbour's boundary record at the
same position.

--iisph runs the scene with the IISPH solver (dt = 1e-3, build_sharded(iisph=True)) and checks the same things as
--dfsph: the pressure sweep count of every step against the single engine's, counts and average errors bit-identical
across ranks in every step, and the ghost alignment; it also reports the per-step average errors of both engines.  The
tolerance rule is test_iisph_steps_vs_oracle's: |dx| / d < 2e-3 when the sweep counts match, 5e-2 otherwise.

--collide splits the fluid into two blocks (objects 0 and 1) that move toward each other at +-vx and meet at the
initial cut of a balanced two-rank start: the fluid along the contact plane is compressed above the rest density within
a few steps, so the pressure solves of DFSPH and IISPH run several sweeps right at the cut.

--dynamic-body / --dynamic-block add dynamic solids (WCSPH, build_sharded(dynamic_solids=True)): a shape-matched cube
(tests/golden/cube.obj) straddling the fluid's x fraction 1/world (1/2 on one rank) -- the initial cut of a balanced
start -- and resting on the fluid surface, and an advected dynamic rigid block on the surface at 3/4 of the fluid.  The tool then also reports whether
every body's cm and R were bit-identical on every rank after every step, whether the fluid's reactions acted (every
dynamic object's mean velocity left free fall, in both engines), and the per-body cm / R differences; "ok" then also
requires max_dv < 1e-2 and per-body |dcm| / d and max |dR| below 1e-3.  --body-vy gives the dynamic solids an initial
vertical velocity (a body thrown into the fluid raises pressures under it within a few steps).

--iisph together with --dynamic-body / --dynamic-block builds with build_sharded(iisph_bodies=True) and reports both
sets: the sweep counts, their equality across ranks and the ghost alignment, and the body and reaction checks.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
EMU = os.environ.get("SPH_EMU_LIB")  # host-emulated library (tests/emu/): CPU tensors, gloo instead of NCCL
if EMU:
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import emu_engine
    emu_engine.install(EMU)
import numpy as np
import torch
import torch.distributed as dist

from sph_taichi_b200 import ParticleSystem, SimConfig, scene, slab


def static_block_scene(c, d):
    """The dam break one spacing above a static floor block (object 1, three lattice layers thick) that spans twice
    the fluid's x extent and its whole z extent: every cut of the fluid also cuts the block, and the fluid slides
    along it."""
    sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * d + 0.2, c[1] * d + 0.4, c[2] * d + 0.12],
                             start=[0.06, 0.10, 0.06])
    lo = [0.04, 0.04, 0.04]
    n = [2 * c[0], 3, c[2] + 2]
    sc["RigidBlocks"] = [{"objectId": 1, "start": lo, "end": [s + (k - 0.5) * d for s, k in zip(lo, n)],
                          "translation": [0.0, 0.0, 0.0], "scale": [1, 1, 1], "velocity": [0.0, 0.0, 0.0],
                          "density": 1000.0, "color": [255, 255, 255], "isDynamic": False}]
    return sc


def colliding_blocks_scene(c, d, vx):
    """The dam break of ``c`` particles split in x into two blocks one lattice spacing apart, the left half (object 0)
    moving at +vx, the right half (object 1) at -vx (--collide)."""
    sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * d + 0.2, c[1] * d + 0.4, c[2] * d + 0.12], start=[0.06] * 3)
    left = sc["FluidBlocks"][0]
    half = c[0] // 2
    right = dict(left, objectId=1, start=[0.06 + half * d] + left["start"][1:], velocity=[-vx, 0.0, 0.0])
    left.update(end=[0.06 + (half - 0.5) * d] + left["end"][1:], velocity=[vx, 0.0, 0.0])
    sc["FluidBlocks"].append(right)
    return sc


def add_dynamic_solids(sc, c, d, world, body, block, vy=0.0):
    """The dynamic solids of --dynamic-body / --dynamic-block on top of the dam break of ``c`` particles (start 0.06),
    with the initial vertical velocity ``vy``."""
    x0, top, z0 = 0.06, 0.06 + c[1] * d, 0.06
    side = 4.5 * d
    if body:
        cut = x0 + c[0] * d / max(world, 2)  # world 1: the middle
        sc.setdefault("RigidBodies", []).append({
            "objectId": 2, "geometryFile": os.path.join(ROOT, "tests", "golden", "cube.obj"),
            "translation": [cut - side / 2, top + 0.25 * d, z0 + (c[2] * d - side) / 2], "rotationAxis": [0, 1, 0],
            "rotationAngle": 0, "scale": [side] * 3, "velocity": [0.0, vy, 0.0], "density": 800.0,
            "color": [255, 255, 255], "isDynamic": True})
    if block:
        bx = x0 + 0.75 * c[0] * d
        sc.setdefault("RigidBlocks", []).append({
            "objectId": 3, "start": [bx, top, z0 + d], "end": [bx + 2.5 * d, top + 2.5 * d, z0 + 3.5 * d],
            "translation": [0.0, 0.0, 0.0], "scale": [1, 1, 1], "velocity": [0.0, vy, 0.0], "density": 600.0,
            "color": [255, 0, 0], "isDynamic": True})
    return sc


def dynamic_velocities(V, OID, FL, g_y, t, vy0=0.0):
    """{object_id: (mean v_y, deviation from free fall)} of the dynamic solids (objects start at v_y = ``vy0``)."""
    out = {}
    dyn = (FL & 3) == 2
    for oid in sorted(set(OID[dyn].tolist())):
        m = dyn & (OID == oid)
        vy = float(V[m][:, 1].double().mean())
        out[int(oid)] = (vy, abs(vy - vy0 - g_y * t))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--counts", type=int, nargs=3, default=[64, 24, 24])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--vx", type=float, default=1.5)
    ap.add_argument("--skew", type=int, default=0, help="shift every interior slab cut by this many layers at the start")
    ap.add_argument("--rebalance-every", type=int, default=8)
    ap.add_argument("--dfsph", action="store_true", help="DFSPH instead of WCSPH (simulationMethod 4, dt = 4e-3)")
    ap.add_argument("--iisph", action="store_true",
                    help="IISPH instead of WCSPH (simulationMethod 3, dt = 1e-3; build_sharded(iisph=True))")
    ap.add_argument("--static-block", action="store_true",
                    help="the fluid rests on a static rigid block that straddles every cut (static_block_scene)")
    ap.add_argument("--collide", action="store_true",
                    help="two fluid blocks meeting at +-vx at the initial cut (colliding_blocks_scene)")
    ap.add_argument("--dynamic-body", action="store_true",
                    help="a shape-matched cube across the initial cut (WCSPH; with --iisph: iisph_bodies=True)")
    ap.add_argument("--dynamic-block", action="store_true",
                    help="an advected dynamic rigid block (WCSPH; with --iisph: iisph_bodies=True)")
    ap.add_argument("--body-vy", type=float, default=0.0, help="initial vertical velocity of the dynamic solids")
    ap.add_argument("--scene", default=None, choices=sorted(scene.NAMED_SCENES),
                    help="a named scene as it is (--counts, --vx and --static-block do not apply; a DFSPH scene needs "
                         "--dfsph for the iteration-count comparison, an IISPH scene --iisph)")
    ap.add_argument("--soak", type=int, default=0, metavar="EVERY",
                    help="long run: read the step state (capacity / out-of-grid flags raise) every EVERY steps; the "
                         "flow is chaotic over thousands of steps, so the verdict is the particle set, finiteness and "
                         "the bulk quantities (centre of mass, kinetic energy) instead of the per-particle distance")
    a = ap.parse_args()
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    dev = torch.device("cpu") if EMU else torch.device(f"cuda:{local}")
    torch.cuda.set_device(dev)
    if world > 1:
        if EMU:
            dist.init_process_group("gloo", rank=rank, world_size=world)
        else:
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    d = 0.02
    c = a.counts
    if a.scene:
        sc = scene.NAMED_SCENES[a.scene]()
        d = 2.0 * sc["Configuration"]["particleRadius"]
    elif a.static_block:
        sc = static_block_scene(c, d)
    elif a.collide:
        sc = colliding_blocks_scene(c, d, a.vx)
    else:
        sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * d + 0.2, c[1] * d + 0.4, c[2] * d + 0.12], start=[0.06] * 3)
    dynamic = a.dynamic_body or a.dynamic_block
    if dynamic and not a.scene:
        sc = add_dynamic_solids(sc, c, d, world, a.dynamic_body, a.dynamic_block, a.body_vy)
    if a.scene and slab.scene_has_dynamic_solids(SimConfig(sc)):
        dynamic = True
    if not a.scene and not a.collide:
        sc["FluidBlocks"][0]["velocity"] = [a.vx, 0.0, 0.0]
    if a.dfsph and sc["Configuration"]["simulationMethod"] != 4:
        sc = scene._as_dfsph(sc)
    if a.iisph and sc["Configuration"]["simulationMethod"] != 3:
        sc = scene._as_iisph(sc)
    jacobi = a.dfsph or a.iisph  # one step per call, sweep counts and the ghost alignment checked
    transport = slab.GlooTransport() if (EMU and world > 1) else None
    slabs = None
    if a.skew:  # deliberately unbalanced start: every interior cut shifted, the balancer has to move them back
        from sph_taichi_b200.scene import assemble_particles
        cfg = SimConfig(sc)
        arrays, _, _, _ = assemble_particles(cfg, 3, d)
        gx = int(np.ceil(np.array(cfg.get_cfg("domainEnd")) / (2 * d)).astype(int)[0])
        hist = np.bincount(slab.layer_of(arrays["x"], 2 * d), minlength=gx)[:gx]
        base = slab.plan_slabs(hist, world)
        cuts = [s_[0] for s_ in base] + [base[-1][1]]
        cuts = [cuts[0]] + [c_ + a.skew for c_ in cuts[1:-1]] + [cuts[-1]]
        slabs = [(cuts[r], cuts[r + 1]) for r in range(world)]
    sim, n_total = slab.build_sharded(sc, rank, world, dev, rebalance_every=a.rebalance_every, slabs=slabs,
                                      transport=transport, dynamic_solids=dynamic, iisph=a.iisph,
                                      iisph_bodies=bool(a.iisph and dynamic))
    first = sim.info()
    trace = []

    def body_trace():
        return [[c_.tobytes().hex(), R_.tobytes().hex()] for c_, R_ in
                (sim.body_state(b) for b in range(len(sim.bodies)))]

    if a.soak:
        done = 0
        while done < a.steps:
            k = min(a.soak, a.steps - done)
            sim.step(k)
            done += k
            i_ = sim.info()  # raises on a capacity / out-of-grid flag
            trace.append((done, i_["owned"], i_["n_live"], i_["x_lo"], i_["x_hi"]))
    elif a.dfsph:
        for _ in range(a.steps):  # one step per call: the iteration counts of every step
            sim.step(1)
            trace.append((sim.last_iterations_v, sim.last_iterations, sim.last_avg_err_v.hex(), sim.last_avg_err.hex()))
    elif a.iisph:
        for _ in range(a.steps):  # one step per call: the sweep counts of every step
            sim.step(1)
            trace.append((sim.last_iterations, sim.last_avg_err.hex()) + ((body_trace(),) if sim.mode.bodies else ()))
    elif sim.mode.bodies:
        for _ in range(a.steps):  # one step per call: the body states of every step
            sim.step(1)
            trace.append(body_trace())
    else:
        sim.step(a.steps)
    last = sim.info()
    gathered = slab.gather_owned(sim)
    meta = {"owned": (first["owned"], last["owned"]), "halo": 64 * last["halo_records_sent"], "trace": trace,
            "slab0": (first["x_lo"], first["x_hi"]), "slab1": (last["x_lo"], last["x_hi"]), "status": last["status"]}
    if jacobi:
        # the x_0 of the ghost layers ([0, own_begin) and [own_end, n_live)) and of the owned records, as the last
        # step's alignment left them (advect and clamp touch owned records only; the sort comes with the next step)
        x0 = sim.record_views()[2][:, :3].cpu().numpy()
        meta["x0_ghost_left"] = x0[:last["own_begin"]].tolist()
        meta["x0_ghost_right"] = x0[last["own_end"]:last["n_live"]].tolist()
        meta["x0_owned"] = x0[last["own_begin"]:last["own_end"]].tolist()
        meta["transport"] = sim.transport_stats()
    if sim.mode.bodies:
        meta["transport"] = sim.transport_stats()
        meta["halo_cap"] = sim.halo_cap
        meta["body_particles"] = sum(b1 - b0 for _, b0, b1, _cm in sim.bodies)
    metas = [None] * world
    if world > 1:
        dist.all_gather_object(metas, meta)
    else:
        metas = [meta]
    ok = True
    if rank == 0:
        ps = ParticleSystem(SimConfig(sc), device=dev)
        s = ps.build_solver(); s.initialize()
        single_counts, single_errs = [], []
        if a.dfsph:
            for _ in range(a.steps):
                s.step(1)
                single_counts.append([s.last_iterations_v, s.last_iterations])
        elif a.iisph:
            for _ in range(a.steps):
                s.step(1)
                single_counts.append([s.last_iterations])
                single_errs.append(float(s.last_avg_density_error))
        else:
            s.step(a.steps)
        bodies = None
        if sim.mode.bodies:
            bodies = {oid: sim.body_state(b) for b, (oid, *_rest) in enumerate(sim.bodies)}
        cmp_ = slab.compare_with_single(gathered, ps, d, bodies=bodies)
        lo_, hi_ = (torch.tensor(sc["Configuration"][k], dtype=torch.float32) for k in ("domainStart", "domainEnd"))
        X_ = gathered[0].cpu()
        cmp_["finite_inside_domain"] = bool(torch.isfinite(X_).all() and (X_ >= lo_).all() and (X_ <= hi_).all())
        X0, OID0 = gathered[2], gathered[3]
        migrated = any(m["owned"][0] != m["owned"][1] for m in metas)
        moved = any(tuple(m["slab0"]) != tuple(m["slab1"]) for m in metas)
        ok = cmp_["same_particle_set"] and cmp_["max_dx_over_d"] < 1e-3 and cmp_["max_dv"] < 1e-2 and slab.static_solids_ok(cmp_)
        solid = ps._t["material"][:n_total] == 0
        if bool(solid.any()):  # [first, last + 1) cell layer the solids occupy
            lay = slab.layer_of(ps._t["x"][:n_total][solid].cpu().numpy(), 2 * d)
            cmp_["solid_layers"] = [int(lay.min()), int(lay.max()) + 1]
        if a.dynamic_body and not a.scene:  # [first, last + 1) cell layer the cube occupies at the start
            lay = slab.layer_of(np.asarray(X0[OID0 == 2].cpu().numpy()), 2 * d)
            cmp_["body_layers"] = [int(lay.min()), int(lay.max()) + 1]
        if jacobi:
            counts = [list(t[:2 if a.dfsph else 1]) for t in metas[0]["trace"]]
            same_on_ranks = all([list(t) for t in m["trace"]] == [list(t) for t in metas[0]["trace"]] for m in metas)
            aligned = True
            for r in range(1, world):  # rank r's left ghosts <-> rank r-1's last owned records, and vice versa
                gl, gr = metas[r]["x0_ghost_left"], metas[r - 1]["x0_ghost_right"]
                aligned = aligned and len(gl) > 0 and len(gr) > 0
                aligned = aligned and gl == metas[r - 1]["x0_owned"][len(metas[r - 1]["x0_owned"]) - len(gl):]
                aligned = aligned and gr == metas[r]["x0_owned"][:len(gr)]
            counts_match = counts == single_counts
            # the rule of test_dfsph_steps_vs_oracle / test_iisph_steps_vs_oracle: tight when the solvers ran the same
            # sweeps
            tol = 2e-3 if counts_match else 5e-2
            ok = (cmp_["same_particle_set"] and cmp_["max_dx_over_d"] < tol and same_on_ranks and aligned
                  and slab.static_solids_ok(cmp_))
            cmp_ = dict(cmp_, iterations_sharded=counts, iterations_single=single_counts, counts_match=counts_match,
                        bit_identical_across_ranks=same_on_ranks, ghosts_aligned=aligned,
                        transport_groups=[m["transport"][0] for m in metas],
                        transport_bytes=[m["transport"][1] for m in metas])
            if a.iisph:
                cmp_.update(avg_err_sharded=[float.fromhex(t[1]) for t in metas[0]["trace"]], avg_err_single=single_errs)
        if sim.mode.bodies:
            same_on_ranks = all(json.dumps(m["trace"]) == json.dumps(metas[0]["trace"]) for m in metas)
            g_y, t = float(sc["Configuration"]["gravitation"][1]), a.steps * float(sc["Configuration"]["timeStepSize"])
            X, V, X0, OID, MV, FL = gathered
            vs = dynamic_velocities(V, OID, FL, g_y, t, a.body_vy)
            ps._pull()
            n_ = int(ps.particle_num[None])
            fl1 = (ps._t["material"][:n_] != 1).int() * 2 * (ps._t["is_dynamic"][:n_] != 0).int()
            v1 = dynamic_velocities(ps._t["v"][:n_], ps._t["object_id"][:n_], fl1, g_y, t, a.body_vy)
            acted = bool(vs) and all(vs[o][1] > 1e-3 and v1[o][1] > 1e-3 for o in vs)
            bodies_ok = all(b["dcm_over_d"] < 1e-3 and b["max_dR"] < 1e-3 for b in cmp_.get("bodies", []))
            ok = (cmp_["same_particle_set"] and cmp_["max_dx_over_d"] < 1e-3 and cmp_["max_dv"] < 1e-2
                  and same_on_ranks and bodies_ok and slab.static_solids_ok(cmp_)
                  and (not jacobi or cmp_["ghosts_aligned"]))
            cmp_ = dict(cmp_, bodies_bit_identical_across_ranks=same_on_ranks, reactions_acted=acted,
                        dynamic_vy_sharded={str(k): v[0] for k, v in vs.items()},
                        dynamic_vy_single={str(k): v[0] for k, v in v1.items()}, free_fall_vy=a.body_vy + g_y * t,
                        n_bodies=len(sim.bodies), transport_groups=[m["transport"][0] for m in metas],
                        transport_bytes=[m["transport"][1] for m in metas], halo_cap=[m["halo_cap"] for m in metas],
                        body_particles=metas[0]["body_particles"])
        if a.soak:
            X, V = gathered[:2]
            ps._pull()
            rx, rv = ps._t["x"], ps._t["v"]
            bulk = {"com_sharded": [round(float(t), 5) for t in X.double().mean(0)],
                    "com_single": [round(float(t), 5) for t in rx.double().mean(0)],
                    "ke_sharded": float((V.double() ** 2).sum()), "ke_single": float((rv.double() ** 2).sum()),
                    "finite": bool(torch.isfinite(X).all() and torch.isfinite(V).all()),
                    "owned_min_max_over_run": [[min(t[1] for t in m["trace"]), max(t[1] for t in m["trace"])] for m in metas],
                    "slab_cuts_seen": [sorted({(t[3], t[4]) for t in m["trace"]}) for m in metas]}
            com_err = max(abs(p_ - q_) for p_, q_ in zip(bulk["com_sharded"], bulk["com_single"])) / d
            ke_rel = abs(bulk["ke_sharded"] - bulk["ke_single"]) / max(bulk["ke_single"], 1e-30)
            bulk["com_err_over_d"] = com_err; bulk["ke_rel_err"] = ke_rel
            ok = cmp_["same_particle_set"] and bulk["finite"] and com_err < 0.1 and ke_rel < 0.05
            cmp_ = dict(cmp_, soak=bulk)
        print(json.dumps(dict(cmp_, world=world, particles=int(n_total), steps=a.steps, migrated=bool(migrated),
                              cuts_moved=bool(moved), owned_first_last=[list(map(int, m["owned"])) for m in metas],
                              slabs_first=[list(m["slab0"]) for m in metas], slabs_last=[list(m["slab1"]) for m in metas],
                              halo_bytes=[int(m["halo"]) for m in metas], status=[int(m["status"]) for m in metas],
                              ok=bool(ok))))
    if world > 1:
        flag = torch.tensor([1 if ok else 0], device=dev)
        dist.broadcast(flag, src=0)
        ok = bool(flag.item())
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
