"""The refusal contract of the library's entry points, on the host-emulated build: every entry point that checks a
context's solver or shard mode is called on a context in every state a user can reach (unsharded WCSPH, DFSPH and
IISPH; sharded fluid + static contexts of each solver, configured and begun; WCSPH and IISPH body contexts, also
switched to DFSPH afterwards; contexts whose transport changed its world size after the configure), and must return the
code and the message of the first condition it fails, in the order below.  The configure entry points are checked
with contexts that fail several of their conditions at once.

A call that passes every check returns SPH_OK: the step entry points are called with nsteps = 0, so nothing past the
checks runs.  A refusal changes nothing but the last error, so the calls of one state share its context; a call that
succeeds and changes the context gets a fresh one.  The one call left out is sph_shard_profile_step on a begun static
WCSPH context whose world changed, which would go on to exchange with a peer that does not exist.

This file is also the launcher of the checks: ``python tests/test_entry_preconditions.py run`` with SPH_EMU_LIB
pointing at the emulated library."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))

OK, E_ARG, E_CAPACITY = 0, -1, -3

STATIC_ONLY = "x-slab sharding supports static solids only"
BODIES_WCSPH = "x-slab sharding of dynamic solids is WCSPH only: the DFSPH pressure sweeps scatter"
IISPH_CONTEXT = "this context is in IISPH mode (sph_set_iisph): it steps with sph_iisph_op"
IISPH_SHARDED = "this IISPH context is sharded: step it with sph_shard_iisph_step"
IISPH_SHARD_STEP = "this context is in IISPH mode (sph_set_iisph): a sharded IISPH context steps with"
IISPH_AFTER_CONFIGURE = "call sph_set_iisph(1) before sph_shard_configure, not on a sharded context"
BODIES_IISPH = "dynamic solids in IISPH are single-GPU unless requested"
IISPH_BODIES_CONTEXT = "sph_shard_configure_iisph_bodies shards the dynamic solids of an IISPH context"
BODIES_FIXED = "the body table of a context configured by sph_shard_configure_bodies is fixed"
NOT_CONFIGURED = "sph_shard_configure was not called"
NOT_BEGUN = "sph_shard_begin was not called"
STALE = "neighbour structure is stale: call sph_neighbor_build first"
STALE_LISTS = "neighbour lists are stale: run sph_neighbor_build and op 0"
NO_DFSPH = "sph_set_dfsph(1) was not called"
NO_IISPH = "sph_set_iisph(1) was not called"
NO_BODY = "rigid body index out of range"
SLAB_RANGE = "slab must lie inside the grid"
GHOST_3 = "dynamic solids need ghost_layers >= 3"
UNIFORM = "x-slab sharding needs a single fluid density"
CAPACITY = "capacity: packed particles + 2 * halo_capacity receive slots exceed n_max"
BODY_CAP = "more rigid bodies than the workspace was sized for"
BODY_RANGE = "rigid body solid-id range out of bounds (pack the whole scene's solid count first)"
REST_CM = "a sharded body needs its rest centre of mass"


class Exact(str):
    """An expected message that must match in full (a shorter one is the prefix of another message)."""


# (solver, shard mode, begun, world changed after configure, sph_set_dfsph(1) after the rest)
STATES = {
    "wcsph": ("W", None, False, False, False),
    "dfsph": ("D", None, False, False, False),
    "iisph": ("I", None, False, False, False),
}
for _s, _name in (("W", "wcsph"), ("D", "dfsph"), ("I", "iisph")):
    STATES[f"static_{_name}"] = (_s, "static", False, False, False)
    STATES[f"static_{_name}_begun"] = (_s, "static", True, False, False)
    STATES[f"static_{_name}_begun_moved"] = (_s, "static", True, True, False)
    STATES[f"static_{_name}_moved"] = (_s, "static", False, True, False)
for _s, _name in (("W", "wcsph"), ("I", "iisph")):
    STATES[f"bodies_{_name}"] = (_s, "bodies", False, False, False)
    STATES[f"bodies_{_name}_begun"] = (_s, "bodies", True, False, False)
    STATES[f"bodies_{_name}_begun_moved"] = (_s, "bodies", True, True, False)
    STATES[f"bodies_{_name}_moved"] = (_s, "bodies", False, True, False)
    STATES[f"bodies_{_name}_begun_to_dfsph"] = (_s, "bodies", True, False, True)
    STATES[f"bodies_{_name}_begun_moved_to_dfsph"] = (_s, "bodies", True, True, True)


def expect(state, entry):
    """(return code, message) of `entry` on a context in `state`; message None: a bare code that leaves the last
    error untouched.  None: the cell is not called."""
    s, shard, begun, moved, to_dfsph = STATES[state]
    if to_dfsph:
        s = "D"
    sharded, bodies = shard is not None, shard == "bodies"

    def shard_step(other_solver, solver, bodies_msg=None, world_msg=None):
        if not sharded:
            return E_ARG, NOT_CONFIGURED
        if s != solver:
            return E_ARG, IISPH_SHARD_STEP if s == "I" else other_solver
        if bodies and bodies_msg:
            return E_ARG, bodies_msg
        if not begun:
            return E_ARG, NOT_BEGUN
        if moved and world_msg:
            return E_ARG, world_msg
        return OK, None

    if entry == "sph_step":
        return {"I": (E_ARG, IISPH_CONTEXT), "D": (E_ARG, "sph_step is the fused WCSPH step; DFSPH is driven through "
                                                          "sph_dfsph_op")}.get(s, (OK, None))
    if entry in ("sph_dfsph_op", "sph_dfsph_solve", "sph_dfsph_step"):
        if s == "I":
            return E_ARG, IISPH_CONTEXT
        if s == "W":
            return E_ARG, Exact(NO_DFSPH)
        if entry == "sph_dfsph_op":
            return E_ARG, STALE
        if entry == "sph_dfsph_solve":
            return E_ARG, STALE_LISTS
        return (E_ARG, "this context is sharded: step it with sph_shard_dfsph_step") if sharded else (OK, None)
    if entry in ("sph_iisph_op", "sph_iisph_solve", "sph_iisph_step", "sph_iisph_read"):
        if s != "I":
            return E_ARG, Exact(NO_IISPH)
        if entry == "sph_iisph_read":
            return OK, None
        if sharded:
            return E_ARG, IISPH_SHARDED
        return {"sph_iisph_op": (E_ARG, STALE), "sph_iisph_solve": (E_ARG, STALE_LISTS)}.get(entry, (OK, None))
    if entry == "sph_shard_step":
        return shard_step("sph_shard_step is the WCSPH step; DFSPH contexts step with sph_shard_dfsph_step", "W",
                          world_msg="the transport's world size changed after sph_shard_configure_bodies: configure "
                                    "again" if bodies else None)
    if entry == "sph_shard_profile_step":
        if sharded and s == "W" and not bodies and begun and moved:
            return None
        return shard_step("sph_shard_profile_step times the WCSPH step", "W",
                          bodies_msg="sph_shard_profile_step times the static-solid WCSPH step, not the step of a "
                                     "context configured by sph_shard_configure_bodies")
    if entry == "sph_shard_dfsph_step":
        return shard_step("sph_set_dfsph(1) was not called: WCSPH contexts step with sph_shard_step", "D",
                          bodies_msg=BODIES_WCSPH,
                          world_msg="the transport's world size changed after sph_shard_configure: configure again")
    if entry == "sph_shard_iisph_step":
        return shard_step("sph_set_iisph(1) was not called before sph_shard_configure", "I",
                          world_msg="the transport's world size changed after sph_shard_configure: configure again")
    if entry in ("sph_shard_step(-1)", "sph_shard_dfsph_step(io=NULL)", "sph_shard_iisph_step(-1)",
                 "sph_shard_profile_step(NULL)", "sph_shard_info(NULL)"):
        return (E_ARG, None) if sharded else (E_ARG, NOT_CONFIGURED)
    if entry in ("sph_shard_begin", "sph_halo_exchange", "sph_shard_dump"):
        return (E_ARG, NOT_CONFIGURED) if not sharded else None
    if entry == "sph_shard_info":
        return (E_ARG, NOT_CONFIGURED) if not sharded else (OK, None)
    if entry in ("sph_step(-1)", "sph_dfsph_solve(mode=2)", "sph_dfsph_step(-1)", "sph_iisph_solve(max_iterations=0)",
                 "sph_iisph_step(-1)"):
        return E_ARG, None
    if entry == "sph_set_iisph(1)":
        return (E_ARG, IISPH_AFTER_CONFIGURE) if sharded else (OK, None)
    if entry == "sph_set_iisph(0)":
        return OK, None
    if entry == "sph_set_solid_count(9, dynamic)":
        return E_CAPACITY, "n_solid exceeds the capacity given at creation"
    if entry == "sph_set_solid_count(1, dynamic)":
        return (E_ARG, STATIC_ONLY) if sharded else (OK, None)
    if entry in ("sph_set_solid_count(1, static)", "sph_set_solid_count(0, dynamic)"):
        return OK, None
    if entry == "sph_boundary_volume":
        return (E_ARG, STATIC_ONLY) if sharded else (E_ARG, STALE)
    if entry in ("sph_compute_com", "sph_compute_rigid_rest_cm", "sph_solve_constraints"):
        return (E_ARG, STATIC_ONLY) if sharded else (E_ARG, NO_BODY)
    if entry == "sph_set_rigid_bodies(2)":
        return E_CAPACITY, BODY_CAP
    if entry == "sph_set_rigid_bodies(1)":
        return (E_ARG, STATIC_ONLY) if sharded else (OK, None)
    if entry == "sph_set_rigid_bodies(0)":
        return (E_ARG, BODIES_FIXED) if bodies else (OK, None)
    raise KeyError(entry)


ENTRIES = [
    "sph_step", "sph_dfsph_op", "sph_dfsph_solve", "sph_dfsph_step", "sph_iisph_op", "sph_iisph_solve",
    "sph_iisph_step", "sph_iisph_read", "sph_shard_step", "sph_shard_profile_step", "sph_shard_dfsph_step",
    "sph_shard_iisph_step", "sph_shard_step(-1)", "sph_shard_dfsph_step(io=NULL)", "sph_shard_iisph_step(-1)",
    "sph_shard_profile_step(NULL)", "sph_shard_info(NULL)", "sph_shard_begin", "sph_halo_exchange", "sph_shard_dump",
    "sph_shard_info", "sph_step(-1)", "sph_dfsph_solve(mode=2)", "sph_dfsph_step(-1)",
    "sph_iisph_solve(max_iterations=0)", "sph_iisph_step(-1)", "sph_set_iisph(1)", "sph_set_iisph(0)",
    "sph_set_solid_count(9, dynamic)", "sph_set_solid_count(1, dynamic)", "sph_set_solid_count(1, static)",
    "sph_set_solid_count(0, dynamic)", "sph_boundary_volume", "sph_compute_com", "sph_compute_rigid_rest_cm",
    "sph_solve_constraints", "sph_set_rigid_bodies(2)", "sph_set_rigid_bodies(1)", "sph_set_rigid_bodies(0)",
]

# The configure entry points on unsharded contexts that fail several conditions at once: (name, solver, context
# changes, call, expected code, expected message).  Context changes: "dynamic" (one dynamic solid), "body" (a rigid
# body table), "nonuniform" (fluid masses differ).  Call: (entry point, x_hi - grid width, ghost_layers,
# halo_capacity in units of the packed count, rebalance_every, bodies).
NAN = float("nan")
CONFIGURE = [
    ("range: ghost_layers < 1", "W", ("dynamic", "nonuniform"), ("plain", 0, 0, 1, -1, None), E_ARG, SLAB_RANGE),
    ("range: wider than the grid", "W", ("dynamic",), ("plain", 1, 1, 1, 0, None), E_ARG, SLAB_RANGE),
    ("dynamic solids", "W", ("dynamic", "nonuniform"), ("plain", 0, 1, 2, -1, None), E_ARG, STATIC_ONLY),
    ("a body table", "D", ("body", "nonuniform"), ("plain", 0, 1, 2, 0, None), E_ARG, STATIC_ONLY),
    ("non-uniform fluid", "I", ("nonuniform",), ("plain", 0, 1, 2, -1, None), E_ARG, UNIFORM),
    ("capacity", "W", (), ("plain", 0, 1, 2, -1, None), E_CAPACITY, CAPACITY),
    ("rebalance_every < 0", "D", (), ("plain", 0, 1, 1, -1, None), E_ARG, None),
    ("configured", "I", (), ("plain", 0, 1, 1, 0, None), OK, None),
    ("bodies: n_bodies < 0", "I", (), ("bodies", 1, 0, 2, -1, -1), E_ARG, None),
    ("bodies: IISPH context", "I", ("nonuniform",), ("bodies", 1, 0, 2, -1, []), E_ARG, BODIES_IISPH),
    ("iisph bodies: WCSPH context", "W", (), ("iisph_bodies", 1, 0, 2, -1, []), E_ARG, IISPH_BODIES_CONTEXT),
    ("iisph bodies: DFSPH context", "D", (), ("iisph_bodies", 1, 0, 2, -1, []), E_ARG, IISPH_BODIES_CONTEXT),
    ("bodies: range", "D", ("nonuniform",), ("bodies", 1, 0, 2, -1, []), E_ARG, SLAB_RANGE),
    ("bodies: range before ghost_layers", "W", (), ("bodies", 1, 2, 1, 0, []), E_ARG, SLAB_RANGE),
    ("bodies: ghost_layers 0 is not a range error", "W", ("nonuniform",), ("bodies", 0, 0, 1, 0, []), E_ARG, GHOST_3),
    ("bodies: ghost_layers before DFSPH", "D", (), ("bodies", 0, 2, 1, 0, []), E_ARG, GHOST_3),
    ("bodies: DFSPH context", "D", ("nonuniform",), ("bodies", 0, 3, 2, -1, []), E_ARG, BODIES_WCSPH),
    ("bodies: non-uniform fluid", "W", ("nonuniform",), ("bodies", 0, 3, 2, -1, []), E_ARG, UNIFORM),
    ("iisph bodies: non-uniform fluid", "I", ("nonuniform",), ("iisph_bodies", 0, 3, 2, -1, []), E_ARG, UNIFORM),
    ("bodies: capacity", "W", (), ("bodies", 0, 3, 2, -1, [(1, 0, 5, 0.0)] * 2), E_CAPACITY, CAPACITY),
    ("bodies: rebalance_every < 0", "I", (), ("iisph_bodies", 0, 3, 1, -1, [(1, 0, 5, 0.0)] * 2), E_ARG, None),
    ("bodies: body capacity", "W", (), ("bodies", 0, 3, 1, 0, [(1, 0, 5, NAN)] * 2), E_CAPACITY, BODY_CAP),
    ("bodies: body range", "W", (), ("bodies", 0, 3, 1, 0, [(1, 0, 5, NAN)]), E_ARG, BODY_RANGE),
    ("bodies: rest_cm", "I", (), ("iisph_bodies", 0, 3, 1, 0, [(1, 0, 0, NAN)]), E_ARG, REST_CM),
    ("bodies: configured", "W", (), ("bodies", 0, 3, 1, 0, [(1, 0, 0, 0.0)]), OK, None),
    ("iisph bodies: configured", "I", (), ("iisph_bodies", 0, 3, 1, 0, [(1, 0, 0, 0.0)]), OK, None),
]


# entry points that change the context when they succeed
MUTATING = {"sph_set_iisph(1)", "sph_set_iisph(0)", "sph_set_solid_count(1, dynamic)", "sph_set_solid_count(1, static)",
            "sph_set_solid_count(0, dynamic)", "sph_set_rigid_bodies(1)", "sph_set_rigid_bodies(0)",
            "sph_shard_profile_step"}


def _check(got, want, before=""):
    rc, msg = got
    code, text = want
    if rc != code:
        return False
    if text is None:
        return rc == OK or msg == before  # a bare code leaves the last error as it was
    return msg == text if isinstance(text, Exact) else text in msg


def run_checks():
    import ctypes as C

    import emu_engine
    emu_engine.install(os.environ["SPH_EMU_LIB"])
    import numpy as np
    import torch
    from sph_taichi_b200 import SimConfig, _lib, engine, scene, slab

    cpu = torch.device("cpu")
    cfg = SimConfig(scene.dam_break_box([6, 4, 4], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3))
    params = slab.scene_params(cfg)
    gx = int(params.grid_num[0])
    arrays, _, _, counts = scene.assemble_particles(cfg, 3, 0.02)
    n = counts["total"]
    m_V0 = float(np.float32(0.8 * 0.02 ** 3))
    transport_calls = []

    def refuse(*_):  # the transport a changed world size brings: no entry point here may reach it
        transport_calls.append(1)
        return 1

    cb = (_lib.TRANSPORT_GROUP_START(refuse), _lib.TRANSPORT_GROUP_END(refuse), _lib.TRANSPORT_SEND(refuse),
          _lib.TRANSPORT_RECV(refuse))
    moved_transport = _lib.SphTransport(None, *cb)

    def table(bodies):
        t = (_lib.SphRigidBody * max(1, len(bodies)))()
        for i, (oid, b0, b1, cm) in enumerate(bodies):
            t[i].object_id, t[i].solid_begin, t[i].solid_end = oid, b0, b1
            t[i].rest_cm = (C.c_float * 3)(cm, cm, cm)
        return t

    def fresh(solver, changes=()):
        e = engine.Engine(params, n_max=4 * n, n_solid=8, n_bodies=1, device=cpu)
        e.pack(slab.field_tensors(arrays, n, m_V0, cpu), n, 0, False)
        lib, ctx = e.lib, e.ctx
        if solver == "D":
            assert lib.sph_set_dfsph(ctx, 1) == OK
        if solver == "I":
            assert lib.sph_set_iisph(ctx, 1) == OK
        if "dynamic" in changes:
            assert lib.sph_set_solid_count(ctx, 1, 1) == OK
        if "body" in changes:
            assert lib.sph_set_rigid_bodies(ctx, table([(1, 0, 0, 0.0)]), 1) == OK
        if "nonuniform" in changes:
            assert lib.sph_set_fluid_uniform(ctx, 0, 0.0, 0.0) == OK
        return e

    def state(name):
        solver, shard, begun, moved, to_dfsph = STATES[name]
        e = fresh(solver)
        lib, ctx = e.lib, e.ctx
        if shard == "static":
            assert lib.sph_shard_configure(ctx, 0, gx, 1, n, 0) == OK, lib.sph_last_error(ctx)
        elif shard == "bodies":
            fn = lib.sph_shard_configure_iisph_bodies if solver == "I" else lib.sph_shard_configure_bodies
            assert fn(ctx, 0, gx, 3, n, 0, None, 0) == OK, lib.sph_last_error(ctx)
        if begun:
            assert lib.sph_shard_begin(ctx, None) == OK, lib.sph_last_error(ctx)
        if moved:
            assert lib.sph_comm_set_transport(ctx, C.byref(moved_transport), 0, 2) == OK
        if to_dfsph:
            assert lib.sph_set_dfsph(ctx, 1) == OK
        return e

    dio = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
    iio = _lib.SphIisphStep(max_iterations=1, omega=0.5, eta=1e-3, n_fluid=1, first_batch=1)
    out = torch.zeros(64, dtype=torch.float32)
    ms6 = (C.c_float * 6)()
    info16 = (C.c_int32 * 16)()
    rows, status = C.c_int64(0), C.c_uint32(0)
    calls = {
        "sph_step": lambda L, c: L.sph_step(c, 0, None),
        "sph_dfsph_op": lambda L, c: L.sph_dfsph_op(c, 0, 0.0, None, None),
        "sph_dfsph_solve": lambda L, c: L.sph_dfsph_solve(c, 1, 1, 1e-3, 0.0, 1, 1, None, None, None, None),
        "sph_dfsph_step": lambda L, c: L.sph_dfsph_step(c, 0, C.byref(dio), None),
        "sph_iisph_op": lambda L, c: L.sph_iisph_op(c, 0, 0.0, None, None),
        "sph_iisph_solve": lambda L, c: L.sph_iisph_solve(c, 1, 0.5, 1e-3, 1, 1, None, None, None),
        "sph_iisph_step": lambda L, c: L.sph_iisph_step(c, 0, C.byref(iio), None),
        "sph_iisph_read": lambda L, c: L.sph_iisph_read(c, None, None, None, None),
        "sph_shard_step": lambda L, c: L.sph_shard_step(c, 0, None),
        "sph_shard_profile_step": lambda L, c: L.sph_shard_profile_step(c, ms6, None),
        "sph_shard_dfsph_step": lambda L, c: L.sph_shard_dfsph_step(c, 0, C.byref(dio), None),
        "sph_shard_iisph_step": lambda L, c: L.sph_shard_iisph_step(c, 0, C.byref(iio), None),
        "sph_shard_step(-1)": lambda L, c: L.sph_shard_step(c, -1, None),
        "sph_shard_dfsph_step(io=NULL)": lambda L, c: L.sph_shard_dfsph_step(c, 0, None, None),
        "sph_shard_iisph_step(-1)": lambda L, c: L.sph_shard_iisph_step(c, -1, C.byref(iio), None),
        "sph_shard_profile_step(NULL)": lambda L, c: L.sph_shard_profile_step(c, None, None),
        "sph_shard_info(NULL)": lambda L, c: L.sph_shard_info(c, None, None, None),
        "sph_shard_begin": lambda L, c: L.sph_shard_begin(c, None),
        "sph_halo_exchange": lambda L, c: L.sph_halo_exchange(c, None),
        "sph_shard_dump": lambda L, c: L.sph_shard_dump(c, 0, out.data_ptr(), out.data_ptr(), 0, C.byref(rows),
                                                        C.byref(status), None),
        "sph_shard_info": lambda L, c: L.sph_shard_info(c, info16, None, None),
        "sph_step(-1)": lambda L, c: L.sph_step(c, -1, None),
        "sph_dfsph_solve(mode=2)": lambda L, c: L.sph_dfsph_solve(c, 2, 1, 1e-3, 0.0, 1, 1, None, None, None, None),
        "sph_dfsph_step(-1)": lambda L, c: L.sph_dfsph_step(c, -1, C.byref(dio), None),
        "sph_iisph_solve(max_iterations=0)": lambda L, c: L.sph_iisph_solve(c, 0, 0.5, 1e-3, 1, 1, None, None, None),
        "sph_iisph_step(-1)": lambda L, c: L.sph_iisph_step(c, -1, C.byref(iio), None),
        "sph_set_iisph(1)": lambda L, c: L.sph_set_iisph(c, 1),
        "sph_set_iisph(0)": lambda L, c: L.sph_set_iisph(c, 0),
        "sph_set_solid_count(9, dynamic)": lambda L, c: L.sph_set_solid_count(c, 9, 1),
        "sph_set_solid_count(1, dynamic)": lambda L, c: L.sph_set_solid_count(c, 1, 1),
        "sph_set_solid_count(1, static)": lambda L, c: L.sph_set_solid_count(c, 1, 0),
        "sph_set_solid_count(0, dynamic)": lambda L, c: L.sph_set_solid_count(c, 0, 1),
        "sph_boundary_volume": lambda L, c: L.sph_boundary_volume(c, 1, None),
        "sph_compute_com": lambda L, c: L.sph_compute_com(c, 0, out.data_ptr(), None),
        "sph_compute_rigid_rest_cm": lambda L, c: L.sph_compute_rigid_rest_cm(c, 0, None),
        "sph_solve_constraints": lambda L, c: L.sph_solve_constraints(c, 0, out.data_ptr(), None),
        "sph_set_rigid_bodies(2)": lambda L, c: L.sph_set_rigid_bodies(c, table([(1, 0, 0, 0.0)] * 2), 2),
        "sph_set_rigid_bodies(1)": lambda L, c: L.sph_set_rigid_bodies(c, table([(1, 0, 0, 0.0)]), 1),
        "sph_set_rigid_bodies(0)": lambda L, c: L.sph_set_rigid_bodies(c, None, 0),
    }
    assert set(calls) == set(ENTRIES)
    bad, cells = [], 0
    for name in STATES:
        shared = state(name)
        for entry in ENTRIES:
            want = expect(name, entry)
            if want is None:
                continue
            e = state(name) if want[0] == OK and entry in MUTATING else shared
            before = e.lib.sph_last_error(e.ctx).decode()
            rc = calls[entry](e.lib, e.ctx)
            got = (rc, e.lib.sph_last_error(e.ctx).decode())
            if e is not shared:
                e.close()
            cells += 1
            if not _check(got, want, before):
                bad.append(f"{name} / {entry}: got {got}, want {want}")
        shared.close()
    # the world-size check: no call above reached the transport of a changed world
    if transport_calls:
        bad.append(f"the transport was called {len(transport_calls)} times")
    for what, solver, changes, (fn, over, ghost, halo, rebalance, bodies), code, text in CONFIGURE:
        e = fresh(solver, changes)
        lib, ctx = e.lib, e.ctx
        halo_cap = 2 * n if halo == 2 else n
        if fn == "plain":
            rc = lib.sph_shard_configure(ctx, 0, gx + over, ghost, halo_cap, rebalance)
        else:
            f = lib.sph_shard_configure_iisph_bodies if fn == "iisph_bodies" else lib.sph_shard_configure_bodies
            nb = bodies if isinstance(bodies, int) else len(bodies)
            rc = f(ctx, 0, gx + over, ghost, halo_cap, rebalance, None if isinstance(bodies, int) else table(bodies), nb)
        got = (rc, lib.sph_last_error(ctx).decode())
        cells += 1
        if not _check(got, (code, text)):
            bad.append(f"{what}: got {got}, want {(code, text)}")
        e.close()
    # a refused sph_shard_configure_bodies keeps the context's body table
    e = fresh("W", ("body",))
    lib, ctx = e.lib, e.ctx
    rc = lib.sph_shard_configure_bodies(ctx, 0, gx, 3, n, 0, table([(1, 0, 5, 0.0)]), 1)
    if rc != E_ARG or lib.sph_compute_rigid_rest_cm(ctx, 0, None) != OK:
        bad.append("a refused sph_shard_configure_bodies lost the body table")
    e.close()
    cells += 1
    for line in bad:
        print(line)
    print(f"{cells} cells, {len(bad)} wrong")
    return 1 if bad else 0


def test_every_entry_point_refuses_with_the_first_failed_condition():
    import build_emu
    env = dict(os.environ, SPH_EMU_LIB=build_emu.build(), PYTHONPATH=ROOT)
    env.pop("SPH_B200_LIB", None)
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "run"], capture_output=True, text=True,
                         timeout=1500, env=env, cwd=ROOT)
    tail = res.stdout[-6000:] + res.stderr[-3000:]
    assert res.returncode == 0 and ", 0 wrong" in res.stdout, tail
    cells = int(res.stdout.split(" cells,")[0].split()[-1])
    assert cells > 900, tail


if __name__ == "__main__":
    if sys.argv[1:] != ["run"]:
        sys.exit("usage: test_entry_preconditions.py run")
    sys.exit(run_checks())
