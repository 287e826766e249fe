"""x-slab sharding of one WCSPH, DFSPH, IISPH or PCISPH scene across the GPUs of a node (one process per GPU).

The reference is single-device; this is the multi-GPU extension BASELINE.json asks for (SURVEY.md section 8e).

* The grid is cut into slabs of whole x cell-layers, balanced by particle count (``plan_slabs``).  After the
  counting sort (x-major flattening, reference ``particle_system.py:292-294``) every cell layer is ONE contiguous
  index range of the packed arrays.
* Interaction radius = one cell, so each rank keeps 2 ghost layers per side: densities of the first ghost layer are
  recomputed locally from the second, and a SINGLE exchange per step is enough.
* The whole sharded step lives in ``libsph_b200.so`` (``sph_shard_*``, include/sph_b200.h): live counts, slab
  bounds, send / receive ranges and the record counts (in-band headers) are DEVICE state, the exchange is NCCL
  point-to-point issued by the library on its own communicator, and classify + sort + pair passes + exchange are a
  fixed launch sequence (asynchronous launches by default, one captured CUDA graph per step with
  ``SPH_SHARD_GRAPH=1``).  The host (this module) only builds the scene, hands the library its share and launches
  steps; it never waits on the device inside a step.  Cuts are re-balanced on the device every
  ``rebalance_every`` steps.
* DFSPH scenes (``simulationMethod: 4``) step through ``sph_shard_dfsph_step``: the same sort, re-balancing and
  record exchange, plus a once-per-step ghost alignment and two small exchanges of the outermost owned layer per
  Jacobi sweep; the loops' error sums are all-gathered and added in rank order, so every rank runs the same sweeps.
  That step waits on the host once per batch of sweeps, like the single-GPU DFSPH step, and is always launched
  eagerly: ``SPH_SHARD_GRAPH`` does not apply to it.
* Static solids (``RigidBlocks`` / ``RigidBodies`` with ``isDynamic: false``) ride the record exchange like fluid
  particles and never change.  Their boundary volumes depend on solid neighbours that may sit across a cut, so
  ``build_sharded`` computes them once, before the first exchange, over the whole scene exactly as the single engine
  does (``startup_state``).
* Dynamic solids (shape-matched ``RigidBodies`` and advected ``RigidBlocks`` with ``isDynamic: true``) are opt-in,
  WCSPH only: ``build_sharded(..., dynamic_solids=True)`` configures the engine with ``sph_shard_configure_bodies``.
  Each rank then keeps 3 ghost layers (a moving solid's boundary volume in the second ghost layer sums solids of the
  third), gathers the fluid's reactions onto the dynamic solids it owns (fluid owned across a cut included), and
  solves every body on every rank with the single engine's shape-matching reduction over an all-gather of all body
  particles' records: cm and R are bit-identical on every rank and equal to the single engine's for the same particle
  positions (``ShardedSimulation.body_state``).  The bodies' rest centres of mass are computed over the whole scene
  exactly as the single engine computes them, in the same pass as the boundary volumes (``startup_state``).  That
  step is launched eagerly, without overlap; ``SPH_SHARD_GRAPH`` does not apply.  Without the flag, and for DFSPH in
  any case, dynamic solids are refused (``STATIC_SOLIDS_ONLY`` / ``DYNAMIC_SOLIDS_WCSPH_ONLY``): the DFSPH pressure
  sweeps scatter the reactions in every sweep, which would need a reaction exchange per sweep.
* IISPH scenes (``simulationMethod: 3``) are opt-in: ``build_sharded(..., iisph=True)`` (``run_simulation.py --gpus N
  --shard-iisph``); without it they are refused (``IISPH_SINGLE_GPU``).  They step through ``sph_shard_iisph_step``,
  the DFSPH step's shape with IISPH's substep: the once-per-step ghost alignment, the predicted velocities and the
  warm-start pressures of the outermost owned layer sent once per step, and two small exchanges per relaxed Jacobi
  sweep (its pressure accelerations, then its new pressures); the error sums are added in rank order, so every rank
  runs the same sweeps (``last_iterations`` / ``last_avg_err``).  Dynamic solids in IISPH are a second opt-in,
  ``build_sharded(..., iisph_bodies=True)`` (``--gpus N --shard-iisph-bodies``, ``sph_shard_configure_iisph_bodies``);
  with ``iisph=True`` alone they are refused (``DYNAMIC_SOLIDS_IISPH``).  IISPH scatters the reactions once per step,
  after the pressure loop, so the WCSPH pieces carry over: 3 ghost layers with moving boundary volumes, the final
  pressure acceleration without the scatter, one more message with the first ghost layer's final pressures, the
  reactions gathered onto the owned dynamic solids, and the bodies solved on every rank from the all-gather.  Whether the sharded step beats one GPU at a given scene size depends
  on the sweep count: each sweep costs two transport groups and each batch of sweeps one host wait.
* Sharded PCISPH: PCISPH scenes (``simulationMethod: 1``) are opt-in too: ``build_sharded(..., pcisph=True)``
  (``run_simulation.py --gpus N --shard-pcisph``); without it they are refused (``PCISPH_SINGLE_GPU``).  They step
  through ``sph_shard_pcisph_step``, the DFSPH step's shape with PCISPH's substep: the once-per-step ghost alignment and
  two small exchanges per prediction-correction sweep (the predicted positions {x*, m_V}, then the new pressures) and
  none outside the loop.  The sweep's error is the max of the ranks' partials, which is exact and independent of the
  order, so every rank runs the same sweeps and reports bit-identical ``last_iterations`` /
  ``last_max_density_error``.  Fluid and static solids only: dynamic solids in PCISPH are refused
  (``DYNAMIC_SOLIDS_PCISPH``).
* Output: ``ShardedSimulation.dump(obj_id)`` is ``ParticleSystem.dump`` of a sharded run.  It is collective: every rank
  compacts x and v of that object's owned records on the device and rank 0 receives them over the engine's own
  transport (``sph_shard_dump``), in the global cell order of the last sort.  ``run_simulation.py --gpus N`` writes
  the PLY series and the posed rigid meshes of a sharded run from rank 0 with it; its torch process group (gloo) only
  carries the NCCL id.  ``gather_owned`` stays the parity tools' gather of whole records.

``tests/test_slab_gloo.py`` runs the same library code on the CPU: the host-emulated build of the kernels
(tests/emu/) with ``GlooTransport`` -- torch.distributed point-to-point over gloo -- in place of NCCL.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum
import json
import os
import time

import numpy as np
import torch
import torch.distributed as dist

from . import _lib

GHOST_LAYERS = 2
SEND_LAYERS = GHOST_LAYERS + 2  # one more than the ghost band needs: a cut may move by a layer in any step
GHOST_LAYERS_BODIES = 3  # dynamic solids: moving boundary volumes of the second ghost layer read the third
SEND_LAYERS_BODIES = GHOST_LAYERS_BODIES + 2
RECORD_ARRAYS = 4  # posm, veld, x0id, misc (acc is recomputed every step and not exchanged)
INFO_KEYS = ("n_live", "owned", "x_lo", "x_hi", "step", "own_begin", "own_end", "sendL_begin", "sendL_end",
             "sendR_begin", "sendR_end", "recv_left", "recv_right", "n_sorted", "status")
STATUS_OUT_OF_GRID, STATUS_HALO_CAPACITY, STATUS_SHARD_CAPACITY = 1, 4, 8
STATUS_SHARD_VELOCITY, STATUS_GHOST_ALIGN = 16, 32  # sharded DFSPH (include/sph_b200.h)
STATUS_SOLID_SLOT = 64  # sharded with dynamic solids: two live records with one solid id
FLAG_FLUID, FLAG_DYNAMIC, FLAG_GHOST = 1, 2, 4  # misc.z bits of a packed record (csrc/sph_common.cuh)
STATIC_SOLIDS_ONLY = ("x-slab sharding supports static solids only: dynamic solids (shape-matched bodies, advected "
                      "rigid blocks) are single-GPU in WCSPH and DFSPH")
IISPH_SINGLE_GPU = ("IISPH (simulationMethod 3) is single-GPU unless sharding is requested: x-slab sharding of an "
                    "IISPH scene is opt-in (build_sharded(..., iisph=True), run_simulation.py --gpus N --shard-iisph)")
DYNAMIC_SOLIDS_WCSPH_ONLY = ("x-slab sharding of dynamic solids is WCSPH only: the DFSPH pressure sweeps scatter the "
                             "reactions onto the bodies in every sweep, which would need a reaction exchange per sweep")
DYNAMIC_SOLIDS_IISPH = ("x-slab sharding of dynamic solids is WCSPH only: dynamic solids in IISPH scenes are single-GPU "
                        "unless requested: build_sharded(..., iisph_bodies=True) / run_simulation.py --gpus N "
                        "--shard-iisph-bodies (sharded IISPH otherwise runs fluid and static solids)")
PCISPH_SINGLE_GPU = ("x-slab sharding runs WCSPH (0), DFSPH (4) and IISPH (3) scenes, not simulationMethod 1 unless "
                     "requested: x-slab sharding of a PCISPH scene is opt-in (build_sharded(..., pcisph=True), "
                     "run_simulation.py --gpus N --shard-pcisph)")
DYNAMIC_SOLIDS_PCISPH = ("x-slab sharding of a PCISPH scene runs fluid and static solids: dynamic solids in PCISPH "
                         "scenes are single-GPU")


class Solver(enum.IntEnum):
    """The solvers a scene can shard with, valued by their ``simulationMethod``."""
    WCSPH = 0
    PCISPH = 1
    IISPH = 3
    DFSPH = 4


@dataclasses.dataclass(frozen=True)
class ShardMode:
    """What a sharded run is: its solver, and whether it shards dynamic solids (``bodies``: 3 ghost layers, reactions
    gathered across cuts, bodies solved on every rank)."""
    solver: Solver
    bodies: bool

    @property
    def ghost_layers(self):
        return GHOST_LAYERS_BODIES if self.bodies else GHOST_LAYERS

    @property
    def send_layers(self):
        return SEND_LAYERS_BODIES if self.bodies else SEND_LAYERS


def scene_has_dynamic_solids(cfg):
    """Whether any rigid body or rigid block of the scene is dynamic."""
    return any(o.get("isDynamic") for o in list(cfg.get_rigid_bodies() or []) + list(cfg.get_rigid_blocks() or []))


def shard_mode(method, scene_dynamic, dynamic_solids=False, iisph=False, iisph_bodies=False, pcisph=False):
    """The ``ShardMode`` of ``build_sharded``'s opt-ins on a scene of ``simulationMethod`` ``method`` that has dynamic
    solids or not (``scene_dynamic``); raises when that mode is not sharded.  ``iisph_bodies`` implies ``iisph`` and
    ``dynamic_solids``; ``pcisph`` shards a PCISPH scene without dynamic solids."""
    if iisph_bodies and method != 3:
        raise ValueError(f"iisph_bodies=True shards an IISPH scene (simulationMethod 3) with dynamic solids, not "
                         f"simulationMethod {method}")
    if pcisph and method != 1:
        raise ValueError(f"pcisph=True shards a PCISPH scene (simulationMethod 1), not simulationMethod {method}")
    if method == 3 and not (iisph or iisph_bodies):
        raise NotImplementedError(IISPH_SINGLE_GPU)
    if method == 1 and not pcisph:
        raise NotImplementedError(PCISPH_SINGLE_GPU)
    if method not in (0, 1, 3, 4):
        raise NotImplementedError(f"x-slab sharding runs WCSPH (0), DFSPH (4) and IISPH (3) scenes, not "
                                  f"simulationMethod {method}")
    if iisph and method != 3:
        raise ValueError(f"iisph=True shards an IISPH scene (simulationMethod 3), not simulationMethod {method}")
    if pcisph and (dynamic_solids or scene_dynamic):
        raise NotImplementedError(DYNAMIC_SOLIDS_PCISPH)
    if iisph and not iisph_bodies and (dynamic_solids or scene_dynamic):
        raise NotImplementedError(DYNAMIC_SOLIDS_IISPH)
    bodies = dynamic_solids or iisph_bodies
    if bodies and method == 4:
        raise NotImplementedError(DYNAMIC_SOLIDS_WCSPH_ONLY)
    return ShardMode(Solver(method), bool(bodies))


def scene_geometry(cfg):
    """(h, grid_num, m_V0, domain size) of a scene as ``ParticleSystem`` derives them; m_V0 in float32, the value the
    engine's fields hold."""
    ds = np.array(cfg.get_cfg("domainEnd"), dtype=np.float64) - np.array(cfg.get_cfg("domainStart"))
    radius = cfg.get_cfg("particleRadius")
    h = radius * 4.0
    return h, np.ceil(ds / h).astype(int), np.float32(0.8 * (2 * radius) ** 3), ds


def scene_params(cfg):
    """The engine constants of a scene, as ``ParticleSystem`` derives them before a solver overrides any."""
    from . import engine as _engine
    _, grid_num, _, ds = scene_geometry(cfg)
    return _engine.make_params(3, grid_num, cfg.get_cfg("particleRadius"), cfg.get_cfg("density0"),
                               cfg.get_cfg("stiffness"), cfg.get_cfg("exponent"), cfg.get_cfg("timeStepSize"),
                               cfg.get_cfg("gravitation"), ds)


def solid_ids(arrays):
    """Global solid ids as ``ParticleSystem._prepare_solids`` assigns them: dense, every object's solids contiguous
    (stable order by object id), -1 for fluid particles."""
    solid = np.nonzero(np.asarray(arrays["material"]) == 0)[0]
    sid = np.full(len(arrays["material"]), -1, np.int32)
    order = np.argsort(np.asarray(arrays["object_id"])[solid], kind="stable")
    sid[solid[order]] = np.arange(solid.size, dtype=np.int32)
    return sid


def field_tensors(arrays, n, m_V0, device):
    """The engine's pack fields of ``n`` particles in the reference's layout (``ParticleSystem.add_particles``:
    x_0 = x, m = density * m_V0); ``arrays["m_V"]`` / ``arrays["solid_id"]`` are used when present."""
    def t(a, dt):  # a copy: on a CPU device, an unpack into the fields must not write through to `arrays`
        return torch.from_numpy(np.array(a, dtype=dt)).to(device)

    dens = t(arrays["density"], np.float32)
    m_V = t(arrays["m_V"], np.float32) if "m_V" in arrays else torch.full((n,), m_V0, dtype=torch.float32, device=device)
    return {
        "object_id": t(arrays["object_id"], np.int32), "x": t(arrays["x"], np.float32),
        "x_0": t(arrays["x"], np.float32), "v": t(arrays["v"], np.float32),
        "acceleration": torch.zeros((n, 3), dtype=torch.float32, device=device),
        "m_V": m_V, "m": dens * m_V0,
        "density": dens, "pressure": t(arrays["pressure"], np.float32), "material": t(arrays["material"], np.int32),
        "is_dynamic": t(arrays["is_dynamic"], np.int32), "color": t(arrays["color"], np.int32),
        "grid_ids": None, "solid_id": t(arrays["solid_id"], np.int32) if "solid_id" in arrays else None,
    }


def dynamic_bodies(cfg, arrays):
    """The shape-matched bodies as the single engine registers them (``ParticleSystem._prepare_solids``): every
    dynamic ``RigidBodies`` object in object-id order, with the range of its global solid ids (``solid_ids``).
    Returns [(object_id, solid_begin, solid_end)]."""
    sid, oid = np.asarray(arrays["solid_id"]), np.asarray(arrays["object_id"])
    out = []
    for b in sorted((cfg.get_rigid_bodies() or []), key=lambda b_: b_["objectId"]):
        if not b["isDynamic"]:
            continue
        ids = sid[(oid == b["objectId"]) & (sid >= 0)]
        if ids.size:
            out.append((int(b["objectId"]), int(ids.min()), int(ids.max()) + 1))
    return out


def startup_state(cfg, arrays, bodies, device):
    """The whole scene's start-up state as the single engine's ``SPHBase.initialize()`` leaves it, computed by the
    same kernels on the same packed scene, hence bit-identical to it.  Returns (m_V of every particle, the rest centre
    of mass of each of ``bodies`` [(object_id, solid_begin, solid_end)]).  m_V holds the boundary volumes of
    ``compute_static_boundary_volume`` then ``compute_moving_boundary_volume``; fluid particles keep m_V0.  The rest
    centres of mass are ``compute_rigid_rest_cm``'s, summed in solid-id order.  They do not depend on m_V (a solid's
    mass is m_V0 * density), so computing them first changes neither result.  ``arrays`` must hold ``solid_id`` and at
    least one solid.  Every rank runs this on the whole scene, so every rank holds the same values."""
    from . import engine as _engine
    n = len(arrays["material"])
    sid = np.asarray(arrays["solid_id"])
    solid = sid >= 0
    n_solid = int(solid.sum())
    m_V0 = float(scene_geometry(cfg)[2])
    eng = _engine.Engine(scene_params(cfg), n_max=n, n_solid=n_solid, n_bodies=len(bodies), device=device)
    try:
        f = field_tensors(arrays, n, m_V0, device)
        eng.pack(f, n, n_solid, bool((np.asarray(arrays["is_dynamic"])[solid] != 0).any()))
        if bodies:
            eng.set_rigid_bodies([(o, b0, b1, [np.nan] * 3) for o, b0, b1 in bodies])
        eng.neighbor_build()
        rest_cms = [eng.compute_com(b).cpu().numpy().astype(np.float32) for b in range(len(bodies))]
        eng.boundary_volume(0)
        eng.boundary_volume(1)
        eng.unpack(f)  # sorted order; solid_id maps it back
        got_sid, got_mV = f["solid_id"].cpu().numpy(), f["m_V"].cpu().numpy()
    finally:
        eng.close()
    by_sid = np.empty(n_solid, np.float32)
    s = got_sid >= 0
    by_sid[got_sid[s]] = got_mV[s]
    m_V = np.full(n, np.float32(m_V0), np.float32)
    m_V[solid] = by_sid[sid[solid]]
    return m_V, rest_cms


def plan_slabs(layer_counts, world, min_width=SEND_LAYERS + 1):
    """Cut ``len(layer_counts)`` x cell-layers into ``world`` contiguous slabs with balanced
    particle counts; every slab at least ``min_width`` layers wide.  Returns [(lo, hi)] * world."""
    counts = np.asarray(layer_counts, dtype=np.int64)
    gx = len(counts)
    if gx < world * min_width:
        raise ValueError(f"{gx} cell layers cannot host {world} slabs of >= {min_width} layers")
    cum = np.concatenate([[0], np.cumsum(counts)])
    total = cum[-1]
    cuts = [0]
    for r in range(1, world):
        target = total * r / world
        c = int(np.searchsorted(cum, target, side="left"))
        # keep room for the slabs on both sides
        c = max(c, cuts[-1] + min_width)
        c = min(c, gx - (world - r) * min_width)
        cuts.append(c)
    cuts.append(gx)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def layer_of(x, h):
    """Cell layer of positions (float32 true division, truncation; particle_system.py:287-289)."""
    return (np.asarray(x, dtype=np.float32)[:, 0] / np.float32(h)).astype(np.int32)


def select_owned(arrays, h, lo, hi):
    lay = layer_of(arrays["x"], h)
    m = (lay >= lo) & (lay < hi)
    return {k: v[m] for k, v in arrays.items()}, int(m.sum())


class GlooTransport:
    """SphTransport on torch.distributed point-to-point over HOST memory (TEST transport: the host-emulated
    library keeps its buffers in host memory; the product path is NCCL inside the library)."""

    def __init__(self, group=None):
        self.group = group
        self.reqs = []
        self.keep = []
        self.send_tag, self.recv_tag = {}, {}

        def view(ptr, nbytes):
            buf = (C.c_uint8 * int(nbytes)).from_address(ptr)
            self.keep.append(buf)
            return torch.frombuffer(buf, dtype=torch.uint8)

        def group_start(_user):
            return 0

        def group_end(_user, _stream):
            for r in self.reqs:
                r.wait()
            self.reqs.clear()
            self.keep.clear()
            return 0

        def send(_user, ptr, nbytes, peer, _stream):
            tag = self.send_tag.get(peer, 0)
            self.send_tag[peer] = tag + 1
            self.reqs.append(dist.isend(view(ptr, nbytes), peer, group=self.group, tag=tag % 30000))
            return 0

        def recv(_user, ptr, nbytes, peer, _stream):
            tag = self.recv_tag.get(peer, 0)
            self.recv_tag[peer] = tag + 1
            self.reqs.append(dist.irecv(view(ptr, nbytes), peer, group=self.group, tag=tag % 30000))
            return 0

        self._cb = (_lib.TRANSPORT_GROUP_START(group_start), _lib.TRANSPORT_GROUP_END(group_end),
                    _lib.TRANSPORT_SEND(send), _lib.TRANSPORT_RECV(recv))
        self.struct = _lib.SphTransport(None, *self._cb)


class ShardedSimulation:
    """This rank's share of a sharded scene: a CUDA engine in slab mode + the library's halo exchange."""

    def __init__(self, cfg, mode, mine, n_mine, slabs, rank, world, device, n_cap, halo_cap, uniform_hint, group=None,
                 rebalance_every=8, transport=None, n_fluid=None, n_solid=0, bodies=None):
        """``mode``: the run's ``ShardMode`` (``shard_mode``).  ``mine``: this rank's initial particles (numpy arrays in
        the reference's field layout); with solids also ``solid_id`` (global ids, ``solid_ids``) and ``m_V`` (start-up
        boundary volumes, ``startup_state``).  ``n_solid``: the solid count of the WHOLE scene (sizes the solid-id
        slot map).  ``bodies`` (a mode with bodies): [(object_id, solid_begin, solid_end, rest_cm)] of the whole scene
        (``dynamic_bodies``, ``startup_state``), an empty list for advected rigid blocks only; None otherwise."""
        from . import engine as _engine
        self.cfg, self.mode, self.rank, self.world, self.group = cfg, mode, rank, world, group
        if mode.solver in (Solver.DFSPH, Solver.IISPH) and not n_fluid:
            raise ValueError("a sharded DFSPH or IISPH scene needs n_fluid, the fluid particle count of ALL ranks")
        self.device = torch.device(device)
        self.slabs0 = [tuple(int(v) for v in s_) for s_ in slabs]
        self.h, self.grid_num, m_V0, _ = scene_geometry(cfg)
        self.m_V0 = float(m_V0)
        self.n_cap, self.halo_cap, self.n_solid = int(n_cap), int(halo_cap), int(n_solid)
        self.bodies = None if bodies is None else list(bodies)
        self.eng = _engine.Engine(scene_params(cfg), n_max=self.n_cap, n_solid=self.n_solid,
                                  n_bodies=len(self.bodies or []), device=self.device)
        e = self.eng
        self._load(mine, n_mine, uniform_hint)
        self.last_iterations_v = self.last_iterations = 0
        self._io = None
        self.last_avg_err = self.last_max_density_error = 0.0
        # the solver is set before sph_shard_configure: the library refuses the switch on a sharded context
        if mode.solver is Solver.DFSPH:
            e.set_dfsph(True)
            from .DFSPH import dfsph_step_io
            self._io = dfsph_step_io(float(cfg.get_cfg("timeStepSize")), float(cfg.get_cfg("density0")), n_fluid)
        elif mode.solver is Solver.IISPH:
            e.set_iisph(True)
            from .IISPH import iisph_step_io
            self._io = iisph_step_io(n_fluid)
        elif mode.solver is Solver.PCISPH:
            e.set_pcisph(True)
            from .PCISPH import pcisph_step_io, scaling_factor
            self._io = pcisph_step_io(scaling_factor(cfg.get_cfg("timeStepSize"), cfg.get_cfg("particleRadius")))
        # ---- transport: NCCL inside the library (its own communicator), or a caller-supplied one (tests) ----
        if transport is not None:
            self._transport = transport
            e._check(e.lib.sph_comm_set_transport(e.ctx, C.byref(transport.struct), rank, world), "sph_comm_set_transport")
        elif world > 1:
            ident = [None]
            if rank == 0:
                buf = C.create_string_buffer(128)
                rc = e.lib.sph_comm_unique_id(buf)
                if rc:
                    raise RuntimeError(f"sph_comm_unique_id failed ({rc}): {e.lib.sph_last_error(None).decode()}")
                ident = [buf.raw]
            dist.broadcast_object_list(ident, src=0, group=group)
            e._check(e.lib.sph_comm_init_nccl(e.ctx, ident[0], rank, world), "sph_comm_init_nccl")
        else:
            e._check(e.lib.sph_comm_set_transport(e.ctx, None, 0, 1), "sph_comm_set_transport")
        lo, hi = self.slabs0[rank]
        args = (e.ctx, lo, hi, mode.ghost_layers, self.halo_cap, int(rebalance_every))
        if mode.solver is Solver.PCISPH:
            name = "sph_shard_configure_pcisph"
        elif not mode.bodies:
            name = "sph_shard_configure"
        else:
            table = (_lib.SphRigidBody * max(1, len(self.bodies)))()
            for i, (oid, b0, b1, rest_cm) in enumerate(self.bodies):
                table[i].object_id, table[i].solid_begin, table[i].solid_end = int(oid), int(b0), int(b1)
                table[i].rest_cm = (C.c_float * 3)(*[float(v) for v in rest_cm])
            name = "sph_shard_configure_iisph_bodies" if mode.solver is Solver.IISPH else "sph_shard_configure_bodies"
            args += (table, len(self.bodies))
        e._check(getattr(e.lib, name)(*args), name)
        e._check(e.lib.sph_shard_begin(e.ctx, e._stream()), "sph_shard_begin")
        self.steps_done = 0
        # the scene's objects and per-object particle counts (build_sharded sets them; dump() sizes rank 0's buffers
        # from the counts)
        self.object_collection, self.object_counts = None, None
        self._dump_bufs = None

    def _load(self, arrays, n, uniform_hint):
        """Pack this rank's initial particles (numpy arrays in the reference's field layout)."""
        solid = np.asarray(arrays["material"]) != 1
        if solid.any() and ("solid_id" not in arrays or "m_V" not in arrays):
            raise ValueError("solid particles need their global solid_id and start-up m_V (see build_sharded)")
        f = field_tensors(arrays, n, self.m_V0, self.device)
        self.eng.pack(f, n, self.n_solid, self.mode.bodies, uniform_hint=uniform_hint)
        self.synchronize()  # the temporaries above may be freed now

    @property
    def dfsph(self):
        return self.mode.solver is Solver.DFSPH

    @property
    def iisph(self):
        return self.mode.solver is Solver.IISPH

    @property
    def pcisph(self):
        return self.mode.solver is Solver.PCISPH

    # ---- stepping --------------------------------------------------------------------------------------
    def step(self, n=1):
        """``n`` sharded steps.  DFSPH: ``last_iterations_v`` / ``last_iterations`` (and ``last_avg_err_v`` /
        ``last_avg_err``) are those of the last step, the same on every rank; IISPH: ``last_iterations`` /
        ``last_avg_err`` (pressure sweeps and their last average error), the same on every rank; PCISPH:
        ``last_iterations`` / ``last_max_density_error`` (prediction-correction sweeps and their last max density
        error), the same bits on every rank.  All three wait on the device once per batch of sweeps."""
        e, io = self.eng, self._io
        if self.mode.solver is Solver.DFSPH:
            e._check(e.lib.sph_shard_dfsph_step(e.ctx, int(n), C.byref(io), e._stream()), "sph_shard_dfsph_step")
            self.last_iterations_v, self.last_iterations = int(io.iterations_v), int(io.iterations)
            self.last_avg_err_v, self.last_avg_err = float(io.avg_err_v), float(io.avg_err)
        elif self.mode.solver is Solver.IISPH:  # io.first_batch: in, the previous step's sweeps; out, this step's
            e._check(e.lib.sph_shard_iisph_step(e.ctx, int(n), C.byref(io), e._stream()), "sph_shard_iisph_step")
            self.last_iterations, self.last_avg_err = int(io.iterations), float(io.avg_err)
        elif self.mode.solver is Solver.PCISPH:
            e._check(e.lib.sph_shard_pcisph_step(e.ctx, int(n), C.byref(io), e._stream()), "sph_shard_pcisph_step")
            self.last_iterations, self.last_max_density_error = int(io.iterations), float(io.max_err)
        else:
            e._check(e.lib.sph_shard_step(e.ctx, int(n), e._stream()), "sph_shard_step")
        self.steps_done += int(n)

    def body_state(self, b):
        """(cm [3], R [3, 3]) of body ``b`` (index into ``bodies``) after the last step, as numpy arrays; the same
        bits on every rank."""
        R, cm = self.eng.rigid_state(b)
        return cm, R

    def transport_stats(self):
        """(transport groups issued, bytes this rank sent in them) since the engine was created."""
        out = (C.c_uint64 * 2)()
        e = self.eng
        e._check(e.lib.sph_shard_transport_stats(e.ctx, out), "sph_shard_transport_stats")
        return int(out[0]), int(out[1])

    def profile_step(self):
        """ONE un-graphed step with CUDA events between the stages (synchronises; WCSPH only)."""
        e = self.eng
        buf = (C.c_float * 6)()
        e._check(e.lib.sph_shard_profile_step(e.ctx, buf, e._stream()), "sph_shard_profile_step")
        self.steps_done += 1
        return {"sort_ms": buf[0], "density_boundary_ms": buf[1], "force_boundary_ms": buf[2], "density_interior_ms": buf[3],
                "force_interior_ms": buf[4], "exchange_ms": buf[5]}

    def info(self):
        """The device-resident step state (synchronising read); raises on a capacity / out-of-grid flag."""
        e = self.eng
        out = (C.c_int32 * 16)()
        sent = C.c_uint64(0)
        e._check(e.lib.sph_shard_info(e.ctx, out, C.byref(sent), e._stream()), "sph_shard_info")
        d = {k: int(out[i]) for i, k in enumerate(INFO_KEYS)}
        d["halo_records_sent"] = int(sent.value)
        self._raise_on_status(d["status"], d["n_live"])
        return d

    def _raise_on_status(self, st, n_live):
        """Raise on the flags of a status word (``info``; ``dump`` passes the OR over all ranks)."""
        if st & STATUS_OUT_OF_GRID:
            raise RuntimeError("a particle left the grid (NaN or outside [0, domain))")
        if st & (STATUS_HALO_CAPACITY | STATUS_SHARD_CAPACITY):
            raise RuntimeError(f"rank {self.rank}: slab capacity exceeded (status {st}: halo_capacity {self.halo_cap}, "
                               f"capacity {self.n_cap}{'' if n_live is None else f', live {n_live}'}); "
                               f"raise capacity_factor")
        if st & STATUS_SHARD_VELOCITY:
            raise RuntimeError(f"rank {self.rank}: a particle moved a whole cell layer in x within one step "
                               f"(|v_x| * dt >= h); the record exchange may have lost it -- reduce timeStepSize")
        if st & STATUS_SOLID_SLOT:
            raise RuntimeError(f"rank {self.rank}: two live records carry the same solid id (status {st})")
        if st & STATUS_GHOST_ALIGN:
            raise RuntimeError(f"rank {self.rank}: a neighbour's boundary layers and this rank's ghost layers differ "
                               f"(status {st})")

    def dump(self, obj_id):
        """Collective (call it on every rank between steps with the same ``obj_id``): x and v of object ``obj_id``
        gathered from every rank over the engine's own transport (``sph_shard_dump``).  Rank 0 returns
        ``{"position": [n, 3], "velocity": [n, 3]}`` float32 numpy arrays (the keys of ``ParticleSystem.dump``) in the
        global cell order of the last sort; the other ranks return None.  Every rank sees the OR of all ranks' status
        words and raises on it as ``info()`` does, so all of them raise together."""
        e = self.eng
        if self.rank == 0:
            if not self.object_counts:
                raise ValueError("dump() on rank 0 needs object_counts (set by build_sharded) to size its buffers")
            cap = max(self.object_counts.values())  # rows of the largest object
        else:
            cap = self.n_cap  # at most every record this rank holds
        if self._dump_bufs is None or self._dump_bufs[0].shape[0] != cap:
            self._dump_bufs = tuple(torch.empty((max(cap, 1), 3), dtype=torch.float32, device=self.device)
                                    for _ in range(2))
        x, v = self._dump_bufs
        rows, status = C.c_int64(0), C.c_uint32(0)
        rc = e.lib.sph_shard_dump(e.ctx, int(obj_id), C.c_void_p(x.data_ptr()), C.c_void_p(v.data_ptr()), int(cap),
                                  C.byref(rows), C.byref(status), e._stream())
        e._check(rc, "sph_shard_dump")
        self._raise_on_status(int(status.value), None)
        if self.rank != 0:
            return None
        n = int(rows.value)
        return {"position": x[:n].to("cpu", copy=True).numpy(), "velocity": v[:n].to("cpu", copy=True).numpy()}

    @property
    def slab(self):
        d = self.info()
        return d["x_lo"], d["x_hi"]

    @property
    def halo_bytes(self):
        return 16 * RECORD_ARRAYS * self.info()["halo_records_sent"]

    def owned_count(self):
        return self.info()["owned"]

    def record_views(self):
        """The 4 exchanged packed arrays as [n_cap, 4] float32 views of the engine workspace (current buffer set)."""
        off = (C.c_uint64 * 5)()
        e = self.eng
        e._check(e.lib.sph_state_offsets(e.ctx, off), "sph_state_offsets")
        base = e._ws_ptr - e.workspace.data_ptr()
        views = []
        for k in range(RECORD_ARRAYS):
            b0 = base + int(off[k])
            views.append(e.workspace[b0:b0 + self.n_cap * 16].view(torch.float32).view(self.n_cap, 4))
        return views

    def owned_tensors(self):
        """(x, v, x_0, object_id, m_V, flags) of the owned particles as device tensors ([owned, 3] / [owned]); flags
        holds the record's FLAG_* bits (FLAG_FLUID clear: a solid)."""
        d = self.info()
        v = self.record_views()
        b, e_ = d["own_begin"], d["own_end"]
        flags = v[3][b:e_, 2].contiguous().view(torch.int32)
        keep = (flags & FLAG_GHOST) == 0
        oid = v[2][b:e_, 3].contiguous().view(torch.int32)
        return (v[0][b:e_, :3][keep], v[1][b:e_, :3][keep], v[2][b:e_, :3][keep], oid[keep], v[0][b:e_, 3][keep],
                flags[keep])

    def owned_state(self):
        x, v, x0 = self.owned_tensors()[:3]
        return x.cpu().numpy(), v.cpu().numpy(), x0.cpu().numpy()

    def launch_count(self):
        return self.eng.launch_count()

    def synchronize(self):
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)


def build_sharded(scene_dict, rank, world, device, group=None, capacity_factor=1.2, rebalance_every=8, slabs=None,
                  transport=None, dynamic_solids=False, iisph=False, iisph_bodies=False, pcisph=False):
    """Assemble the scene on every rank, plan the slabs from the initial layer histogram and load this rank's
    share into a CUDA engine.  ``dynamic_solids=True`` opts in to sharding WCSPH scenes with dynamic solids
    (3 ghost layers, reactions gathered across cuts, bodies solved on every rank from an all-gather of their particles).
    ``iisph=True`` opts in to sharding an IISPH scene (fluid and static solids); ``iisph_bodies=True`` to sharding an
    IISPH scene with dynamic solids (it implies ``iisph`` and the layout of ``dynamic_solids``).  ``pcisph=True`` opts
    in to sharding a PCISPH scene (fluid and static solids).
    Returns (ShardedSimulation, n_total)."""
    from .config_builder import SimConfig
    from .scene import assemble_particles

    cfg = SimConfig(scene_dict)
    mode = shard_mode(cfg.get_cfg("simulationMethod"), scene_has_dynamic_solids(cfg), dynamic_solids, iisph,
                      iisph_bodies, pcisph)
    h, grid_num, m_V0, _ = scene_geometry(cfg)
    arrays, object_collection, _, counts = assemble_particles(cfg, 3, 2 * cfg.get_cfg("particleRadius"))
    object_ids, object_sizes = np.unique(arrays["object_id"], return_counts=True)
    gx = int(grid_num[0])
    hist = np.bincount(layer_of(arrays["x"], h), minlength=gx)[:gx]
    if slabs is None:
        slabs = plan_slabs(hist, world, min_width=mode.send_layers + 1)
    fluid = arrays["material"] == 1
    if not mode.bodies and bool((~fluid & (arrays["is_dynamic"] != 0)).any()):
        raise NotImplementedError(STATIC_SOLIDS_ONLY)
    n_solid = int((~fluid).sum())
    table, rest_cms = [], []
    if n_solid:
        arrays["solid_id"] = solid_ids(arrays)
        if mode.bodies:
            table = dynamic_bodies(cfg, arrays)
        arrays["m_V"], rest_cms = startup_state(cfg, arrays, table, device)
    bodies = [t + (cm,) for t, cm in zip(table, rest_cms)] if mode.bodies else None
    lo, hi = slabs[rank]
    mine, n_mine = select_owned(arrays, h, lo, hi)
    # one decision for the whole scene (a rank may start empty), the single engine's: all FLUID particles share m
    # and m_V (solids do not count)?
    m_fluid = arrays["density"][fluid].astype(np.float32) * m_V0
    uniform = bool(m_fluid.size and (m_fluid == m_fluid[0]).all())
    hint = (uniform, float(m_fluid[0]) if m_fluid.size else 0.0, float(m_V0))
    # the fullest layer bounds every layer the front may reach later: SEND_LAYERS of them per side and direction
    halo_cap = int(mode.send_layers * int(hist.max()) * capacity_factor) + 1024
    ghost_est = 2 * mode.ghost_layers * int(hist.max())
    n_cap = int((n_mine + ghost_est) * capacity_factor) + 4 * halo_cap + 1024  # live + trash + 2 receive regions
    sim = ShardedSimulation(cfg, mode, mine, n_mine, slabs, rank, world, device, n_cap, halo_cap, hint, group=group,
                            rebalance_every=rebalance_every, transport=transport, n_fluid=int(fluid.sum()),
                            n_solid=n_solid, bodies=bodies)
    sim.object_collection = object_collection  # the meshes of the OBJ export (restPosition, restCenterOfMass)
    sim.object_counts = {int(o): int(k) for o, k in zip(object_ids, object_sizes)}
    return sim, counts["total"]


# -----------------------------------------------------------------------------------------------
# sharded state against the single-GPU engine (bench.py --gpus N parity_check, tools/check_slab_parity.py)
# -----------------------------------------------------------------------------------------------
def _lexsort_rows(x0, oid=None):
    """Permutation sorting the rows of a [n, 3] tensor lexicographically (x, then y, then z) on its device; with
    ``oid`` the object id is the leading key."""
    order = torch.arange(x0.shape[0], device=x0.device)
    for col in (2, 1, 0):
        _, idx = torch.sort(x0[order, col], stable=True)
        order = order[idx]
    if oid is not None:
        _, idx = torch.sort(oid[order], stable=True)
        order = order[idx]
    return order


def gather_owned(sim, dst=0):
    """All ranks' owned (x, v, x_0, object_id, m_V, flags) gathered on rank `dst` as device tensors (None
    elsewhere)."""
    x, v, x0, oid, m_V, flags = sim.owned_tensors()
    rec = torch.cat([x, v, x0, oid.view(torch.float32)[:, None], m_V[:, None], flags.view(torch.float32)[:, None]],
                    dim=1).contiguous()

    def split(t):
        return (t[:, 0:3], t[:, 3:6], t[:, 6:9], t[:, 9].contiguous().view(torch.int32), t[:, 10].contiguous(),
                t[:, 11].contiguous().view(torch.int32))

    if sim.world == 1:
        return split(rec)
    n = torch.tensor([rec.shape[0]], device=rec.device, dtype=torch.int64)
    counts = [torch.zeros_like(n) for _ in range(sim.world)]
    dist.all_gather(counts, n, group=sim.group)
    counts = [int(c.item()) for c in counts]
    cap = max(counts)
    pad = torch.zeros((cap, rec.shape[1]), device=rec.device, dtype=rec.dtype)
    pad[:rec.shape[0]] = rec
    bufs = [torch.empty_like(pad) for _ in range(sim.world)] if sim.rank == dst else None
    dist.gather(pad, bufs, dst=dst, group=sim.group)
    if sim.rank != dst:
        return None
    return split(torch.cat([b[:c] for b, c in zip(bufs, counts)], dim=0))


def compare_with_single(gathered, ps, d, bodies=None):
    """Rank 0: the gathered sharded state against a ParticleSystem that ran the same steps on ONE GPU, particles
    matched by (object_id, x_0).  With solids in the scene it also reports whether every static solid is still
    exactly at x_0 and the largest relative difference of the static solids' m_V from the single engine's.  With
    dynamic solids: the largest distance of the fluid and of the dynamic solids alone (over d); with ``bodies``
    ({object_id: (cm, R)} of the sharded run) per body |cm - cm_single| / d and max |R - R_single|."""
    X, V, X0, OID, MV, FL = gathered
    ps._pull()
    n = int(ps.particle_num[None])
    rx, rv, rx0, roid, rmv = (ps._t[k][:n] for k in ("x", "v", "x_0", "object_id", "m_V"))
    same = tuple(X0.shape) == tuple(rx0.shape)
    dx = dv = float("inf")
    out = {}
    if same:
        ks, kr = _lexsort_rows(X0, OID), _lexsort_rows(rx0, roid)
        same = bool(torch.equal(X0[ks], rx0[kr]) and torch.equal(OID[ks], roid[kr]))
        if same:
            dx = float((X[ks] - rx[kr]).abs().max().item() / d)
            dv = float((V[ks] - rv[kr]).abs().max().item())
            static = ((FL[ks] & (FLAG_FLUID | FLAG_DYNAMIC)) == 0)
            if bool(static.any()):
                a, b = MV[ks][static].double(), rmv[kr][static].double()
                out = {"static_solids": int(static.sum().item()),
                       "static_solids_at_x0": bool(torch.equal(X[ks][static], X0[ks][static])),
                       "max_rel_dm_V_static": float(((a - b).abs() / b.abs()).max().item())}
            dyn = ((FL[ks] & (FLAG_FLUID | FLAG_DYNAMIC)) == FLAG_DYNAMIC)
            if bool(dyn.any()):
                fl = (FL[ks] & FLAG_FLUID) != 0
                dist_ = (X[ks] - rx[kr]).abs().max(dim=1).values / d
                out["dynamic_solids"] = int(dyn.sum().item())
                out["max_dx_over_d_dynamic_solids"] = float(dist_[dyn].max().item())
                out["max_dx_over_d_fluid"] = float(dist_[fl].max().item()) if bool(fl.any()) else 0.0
    if bodies:
        rows = []
        for oid in sorted(bodies):
            cm, R = (np.asarray(t, np.float64) for t in bodies[oid])
            R1, cm1 = ps._engine.rigid_state(ps._body_index[oid])
            rows.append({"object_id": int(oid), "dcm_over_d": float(np.abs(cm - cm1).max() / d),
                         "max_dR": float(np.abs(R - R1).max())})
        out["bodies"] = rows
    return dict({"same_particle_set": bool(same), "max_dx_over_d": dx, "max_dv": dv, "particles": int(X0.shape[0])},
                **out)


def static_solids_ok(cmp_):
    """The static-solid part of a ``compare_with_single`` result (true without static solids)."""
    return cmp_.get("static_solids_at_x0", True) and cmp_.get("max_rel_dm_V_static", 0.0) < 1e-6


# -----------------------------------------------------------------------------------------------
# bench.py --gpus N (launched by torchrun, one rank per GPU)
# -----------------------------------------------------------------------------------------------
def bench_main(args):
    import bench as _bench  # the repo-root module: shared helpers
    from . import ParticleSystem, SimConfig

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} needs WORLD_SIZE={args.gpus} (launch with torch.distributed.run); "
                         f"got WORLD_SIZE={world}")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29511")
    dev = torch.device(f"cuda:{local}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    name, sc = _bench.scene_for(world, args.scene)
    d = 2.0 * sc["Configuration"]["particleRadius"]
    sim, n_total = build_sharded(sc, rank, world, dev)
    K, W = args.steps, args.warmup

    # ---- parity_check + the same-run single-GPU time: rank 0 steps the SAME scene on one GPU ----
    P = int(os.environ.get("SPH_BENCH_PARITY_STEPS", "20"))
    counts_sharded = []
    if sim.dfsph:  # one step per call: the Jacobi iteration counts of every step
        for _ in range(P):
            sim.step(1)
            counts_sharded.append([sim.last_iterations_v, sim.last_iterations])
    else:
        sim.step(P)
    gathered = gather_owned(sim)
    parity, strong = None, None
    if rank == 0:
        ps = ParticleSystem(SimConfig(sc), device=dev)
        solver = ps.build_solver()
        solver.initialize()
        counts_single = []
        if sim.dfsph:
            for _ in range(P):
                solver.step(1)
                counts_single.append([solver.last_iterations_v, solver.last_iterations])
        else:
            solver.step(P)
        parity = dict(compare_with_single(gathered, ps, d), steps=P, against="the single-GPU engine on rank 0, same scene, "
                      "particles matched by (object_id, x_0)")
        parity["ok"] = bool(parity["same_particle_set"] and parity["max_dx_over_d"] < 1e-3 and static_solids_ok(parity))
        if sim.dfsph:
            # the rule of test_dfsph_steps_vs_oracle: tight when both ran the same sweeps
            same = counts_sharded == counts_single
            parity.update(iterations_sharded=counts_sharded, iterations_single=counts_single, counts_match=same)
            parity["ok"] = bool(parity["same_particle_set"] and parity["max_dx_over_d"] < (2e-3 if same else 5e-2)
                                and static_solids_ok(parity))
        K1 = max(3, min(K, 20))
        solver.step(3)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        solver.step(K1)
        b.record()
        torch.cuda.synchronize()
        strong = {"t1_ms": a.elapsed_time(b) / K1, "t1_steps": K1,
                  "note": "t1: the whole scene on rank 0's GPU alone (other ranks idle), same run, same scene, "
                          "CUDA-graph steps right after the parity steps"}
        del solver, ps, gathered
        torch.cuda.empty_cache()
    flag = torch.tensor([1 if (parity is None or parity["ok"]) else 0], device=dev)
    dist.broadcast(flag, src=0)
    if not bool(flag.item()):
        if rank == 0:
            print(json.dumps({"error": "parity_check failed", "parity_check": parity}))
        dist.destroy_process_group()
        return 3

    sampler = _bench.ClockSampler(local) if rank == 0 else None  # NVML initialised here, well before the timed region
    sim.step(max(W - P, 3))
    sim.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    if sampler:
        sampler.start()
    info0, launches0, xfer0 = sim.info(), sim.launch_count(), sim.transport_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dist.barrier()
    torch.cuda.synchronize()
    iters = []
    a.record()
    if sim.dfsph:
        for _ in range(K):
            sim.step(1)
            iters.append([sim.last_iterations_v, sim.last_iterations])
    else:
        sim.step(K)
    b.record()
    torch.cuda.synchronize()
    dist.barrier()
    xfer1 = sim.transport_stats()
    ms = torch.tensor([a.elapsed_time(b)], device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    info1 = sim.info()
    owned = torch.tensor([info1["owned"], 64 * (info1["halo_records_sent"] - info0["halo_records_sent"]),
                          sim.launch_count() - launches0], device=dev, dtype=torch.float64)
    tot = owned.clone()
    dist.all_reduce(tot, op=dist.ReduceOp.SUM)
    mx = owned.clone()
    dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    clocks = sampler.stop() if sampler else None
    slabs = [None] * world
    dist.all_gather_object(slabs, [info1["x_lo"], info1["x_hi"]])

    xfer = torch.tensor([float(xfer1[0] - xfer0[0]), float(xfer1[1] - xfer0[1])], device=dev, dtype=torch.float64)
    dist.all_reduce(xfer, op=dist.ReduceOp.SUM)
    if sim.dfsph:
        return _bench_dfsph_tail(args, sim, rank, world, local, name, sc, n_total, parity, strong, ms, tot, mx, clocks,
                                 iters, xfer)

    # ---- per-kernel times on every rank: CUDA events between the stages of un-graphed steps ----
    acc = {}
    R = 10
    for _ in range(R):
        for k_, v_ in sim.profile_step().items():
            acc[k_] = acc.get(k_, 0.0) + v_ / R
    live_now = sim.info()
    peak, peak_src = _bench.measured_hbm_peak()
    roof = torch.tensor([acc["density_boundary_ms"] + acc["density_interior_ms"], acc["force_boundary_ms"] + acc["force_interior_ms"],
                         float(live_now["n_live"]), float(live_now["owned"]), acc["sort_ms"], acc["exchange_ms"]],
                        device=dev, dtype=torch.float64)
    roof_max = roof.clone()
    dist.all_reduce(roof_max, op=dist.ReduceOp.MAX)

    # ---- e2e: every step, H2D of the live records' {x, m_V} and {v, rho} words from pinned host
    # memory, the sharded step, and D2H of the same words (what a host-side consumer reads) ----
    Ke = max(3, min(K, 50))
    cap = sim.n_cap
    h_pos = torch.empty((cap, 4), dtype=torch.float32).pin_memory()
    h_vel = torch.empty((cap, 4), dtype=torch.float32).pin_memory()

    def pull():
        n_live = sim.info()["n_live"]
        v = sim.record_views()
        h_pos[:n_live].copy_(v[0][:n_live], non_blocking=True)
        h_vel[:n_live].copy_(v[1][:n_live], non_blocking=True)
        return n_live

    def push(n_live):
        v = sim.record_views()
        v[0][:n_live].copy_(h_pos[:n_live], non_blocking=True)
        v[1][:n_live].copy_(h_vel[:n_live], non_blocking=True)

    n_live = pull()
    torch.cuda.synchronize()
    dist.barrier()
    moved = 0
    t0 = time.perf_counter()
    for _ in range(Ke):
        push(n_live)
        sim.step()
        moved += 32 * n_live
        n_live = pull()
        moved += 32 * n_live
        torch.cuda.current_stream().synchronize()
    e2e_s = torch.tensor([time.perf_counter() - t0], device=dev, dtype=torch.float64)
    dist.all_reduce(e2e_s, op=dist.ReduceOp.MAX)
    moved_t = torch.tensor([float(moved)], device=dev, dtype=torch.float64)
    dist.all_reduce(moved_t, op=dist.ReduceOp.SUM)
    if rank == 0:
        t_ms = float(ms.item())
        val = K / (t_ms * 1e-3)
        halo_per_step = float(tot[1].item()) / K
        strong.update(tN_ms=t_ms / K, speedup=strong["t1_ms"] / (t_ms / K), n_gpus=world)
        d_ms, f_ms = float(roof_max[0].item()), float(roof_max[1].item())
        kernels = []
        for kind, lms, n_part in (("density", d_ms, float(roof_max[2].item())), ("force", f_ms, float(roof_max[3].item()))):
            ach = _bench.ALGO_BYTES[kind] * n_part / (lms * 1e-3) / 1e9
            kernels.append({"kernel": _bench.KERNEL_NAME[kind] + ", slowest rank", "bound": "hbm", "achieved": ach, "peak": peak,
                            "unit": "GB/s", "frac": ach / peak, "traffic": None, "avg_launch_ms": lms,
                            "particles_this_rank": int(n_part),
                            "algorithmic_bytes_per_particle": _bench.ALGO_BYTES[kind]})
        kernels.sort(key=lambda e_: -e_["avg_launch_ms"])
        roofline = dict(kernels[0])
        roofline.update(peak_source=peak_src, kernels=kernels, sort_ms_slowest_rank=float(roof_max[4].item()),
                        exchange_ms_slowest_rank=float(roof_max[5].item()),
                        note="per GPU, slowest rank; CUDA events between the stages of un-graphed sharded steps (10 steps); "
                             "density = boundary + interior launches over owned + first-ghost-layer particles, forces = boundary "
                             "+ interior launches over owned particles (the interior figure includes waiting for the halo "
                             "exchange if it is not hidden behind the interior passes); the pair kernels are fp32-issue / LSU "
                             "bound, not HBM bound (DESIGN.md section 5)")
        line = {
            "metric": _bench.METRIC, "value": val * n_total / 1e6, "unit": _bench.UNIT, "steps_per_s": val,
            "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": t_ms / K, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": _bench.workload_config(name, sc, n_total, n_total),
            "sharding": {"slabs": slabs, "owned_total": int(tot[0].item()), "owned_max_per_rank": int(mx[0].item()),
                         "ghost_layers": GHOST_LAYERS, "halo_capacity_records": sim.halo_cap,
                         "exchange": "one NCCL send/recv group per step issued by libsph_b200.so on its own communicator, "
                                     "overlapped with the interior force pass; no host synchronisation in a step "
                                     "(asynchronous launches; SPH_SHARD_GRAPH=1 replays one CUDA graph per step); "
                                     "cuts re-balanced on the device every 8 steps"},
            "parity_check": parity,
            "strong_scaling": strong,
            "halo": {"bytes_per_step_all_ranks": halo_per_step,
                     "fraction_of_owned_state": halo_per_step / (64.0 * max(tot[0].item(), 1.0))},
            "clocks": clocks,
            "e2e": {"value": Ke / float(e2e_s.item()) * n_total / 1e6, "unit": _bench.UNIT,
                    "steps_per_s": Ke / float(e2e_s.item()), "steps": Ke,
                    "h2d_bytes_per_step": int(moved_t.item() / (2 * Ke)), "d2h_bytes_per_step": int(moved_t.item() / (2 * Ke)),
                    "note": "per rank and step: pinned-host -> device copy of the live records' position and velocity "
                            "words, sharded step (halo exchange inside), device -> pinned-host copy back; max over ranks"},
            "gpu_launches": int(tot[2].item()),
            "roofline": roofline,
            "stage_ms_slowest_rank": {"sort": float(roof_max[4].item()), "density": d_ms, "force": f_ms,
                                      "exchange_on_comm_stream": float(roof_max[5].item())},
            "cpu_baseline": None,
            "notes": "cpu_baseline is reported by the N = 1 run and by --impl reference (bench.py contract)",
        }
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()
    return 0


def _gpu_name_and_power_limit(index):
    """(card name, enforced power limit in W) of GPU `index`, read now (nvidia-smi query; None if unavailable)."""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                              str(index)], capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        return out[0].strip(), float(out[1])
    except Exception:  # noqa: BLE001 - informational only
        return None, None


def _bench_dfsph_tail(args, sim, rank, world, local, name, sc, n_total, parity, strong, ms, tot, mx, clocks, iters,
                      xfer):
    """The bench line of a sharded DFSPH run.  The WCSPH stage profile (sph_shard_profile_step) does not apply; the
    line reports the Jacobi iteration counts of the timed steps and the transport traffic instead."""
    import bench as _bench
    K, W = args.steps, args.warmup
    card, plimit = _gpu_name_and_power_limit(local)
    if rank == 0:
        t_ms = float(ms.item())
        val = K / (t_ms * 1e-3)
        strong.update(tN_ms=t_ms / K, speedup=strong["t1_ms"] / (t_ms / K), n_gpus=world)
        sweeps = [iv + ip for iv, ip in iters]
        line = {
            "metric": _bench.METRIC, "value": val * n_total / 1e6, "unit": _bench.UNIT, "steps_per_s": val,
            "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": t_ms / K, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": _bench.workload_config(name, sc, n_total, n_total),
            "gpu": {"name": card, "power_limit_w": plimit, "read": "nvidia-smi on rank 0, same run"},
            "sharding": {"owned_total": int(tot[0].item()), "owned_max_per_rank": int(mx[0].item()),
                         "ghost_layers": GHOST_LAYERS, "halo_capacity_records": sim.halo_cap,
                         "exchange": "DFSPH: per step one ghost alignment, one record exchange, the exchanges that open "
                                     "the loops and two per Jacobi sweep (NCCL point-to-point issued by libsph_b200.so "
                                     "on the compute stream, not overlapped); eager launches, one host wait per batch "
                                     "of sweeps; cuts re-balanced on the device every 8 steps"},
            "parity_check": parity,
            "strong_scaling": strong,
            "dfsph": {"iterations_per_step": iters, "mean_iterations_per_step": sum(sweeps) / max(len(sweeps), 1),
                      "transport_groups_per_step_all_ranks": float(xfer[0].item()) / K,
                      "transport_bytes_per_step_all_ranks": float(xfer[1].item()) / K},
            "halo": {"record_bytes_per_step_all_ranks": float(tot[1].item()) / K,
                     "note": "records of the end-of-step exchange (64 B each); the transport bytes above count the "
                             "fixed-size messages actually sent, including the per-sweep ones"},
            "clocks": clocks,
            "gpu_launches": int(tot[2].item()),
            "notes": "iterations_per_step = [divergence, pressure] Jacobi iterations of every timed step",
        }
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()
    return 0
