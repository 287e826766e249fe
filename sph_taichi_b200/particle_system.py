"""``ParticleSystem``: the reference's particle container + neighbour search surface
(reference ``particle_system.py:11-495``) as a thin shell over the CUDA engine.

Same constructor, attributes, field names and methods as the reference so that its driver and
solvers read unchanged; the device work behind each method is one C-ABI call
(``include/sph_b200.h``).  Differences, all deliberate and documented in DESIGN.md:

* fields are ``fields.Field`` objects backed by torch CUDA tensors; the authoritative state
  lives in the engine's packed, sorted SoA buffers and is materialised on access;
* ``domain_start`` is honoured exactly as little as in the reference (SURVEY Q1) -- it must be
  the origin, otherwise construction fails loudly instead of silently mis-hashing;
* the sort is the *stable* counting sort (the reference's serial semantics), so results are
  bit-reproducible run to run;
* no CPU path: construction raises if CUDA or ``libsph_b200.so`` is unavailable.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import engine as _engine
from .config_builder import SimConfig
from .fields import Field, ScalarField
from .scene import assemble_particles, cube_particle_count, cube_positions, rigid_body_lattice

_VEC = ("x", "x_0", "v", "acceleration")
_SCAL_F = ("m_V", "m", "density", "pressure")
_SCAL_I = ("object_id", "material", "is_dynamic")
_PACKED = _VEC + _SCAL_F + _SCAL_I + ("color",)


class ParticleSystem:
    def __init__(self, config: SimConfig, GGUI=False, device=None):
        self.cfg = config
        self.GGUI = GGUI

        self.domain_start = np.array(self.cfg.get_cfg("domainStart"))
        self.domain_end = np.array([1.0, 1.0, 1.0])  # never updated by the reference either (Q1)
        self.domian_end = np.array(self.cfg.get_cfg("domainEnd"))  # sic (particle_system.py:20)
        self.domain_size = self.domian_end - self.domain_start
        self.dim = len(self.domain_size)
        assert self.dim > 1
        if self.dim != 3:
            raise NotImplementedError("only 3-D scenes are reachable in the reference (grid_num[2] is hard-coded)")
        if np.any(self.domain_start != 0.0):
            raise ValueError("domainStart must be the origin: the reference never subtracts it when hashing "
                             "or clamping (particle_system.py:289, sph_base.py:155-174)")
        self.simulation_method = self.cfg.get_cfg("simulationMethod")

        self.material_solid = 0
        self.material_fluid = 1

        self.particle_radius = self.cfg.get_cfg("particleRadius")
        self.particle_diameter = 2 * self.particle_radius
        self.support_radius = self.particle_radius * 4.0
        self.m_V0 = 0.8 * self.particle_diameter ** self.dim

        self.grid_size = self.support_radius
        self.grid_num = np.ceil(self.domain_size / self.grid_size).astype(int)
        self.padding = self.grid_size

        if device is None:
            device = f"cuda:{int(os.environ.get('LOCAL_RANK', 0))}" if torch.cuda.is_available() else None
        if device is None:
            raise RuntimeError("sph_taichi_b200 needs a CUDA device (no CPU fallback)")
        self.device = torch.device(device)

        # ---- count and build all particles (particle_system.py:52-83, 148-211) ----
        arrays, self.object_collection, self.object_id_rigid_body, counts = assemble_particles(
            self.cfg, self.dim, self.particle_diameter)
        self.fluid_particle_num = counts["fluid"]
        self.solid_particle_num = counts["solid"]
        # Emitter / dynamic particle count: the reference plans one (TODO at particle_system.py:85-86, FIXME at :324)
        # but sizes every field for the scene's blocks only.  `emitterReserve` (Configuration key, default 0)
        # reserves room for particles added with add_particles / add_cube AFTER initialize(); the neighbour
        # search always works on particle_num[None] <= particle_max_num particles.
        self.emitter_reserve = int(self.cfg.get_cfg("emitterReserve") or 0)
        self.particle_max_num = counts["total"] + self.emitter_reserve
        self.num_rigid_bodies = len(self.cfg.get_rigid_blocks()) + len(self.cfg.get_rigid_bodies())
        self._n_fluid_blocks = len(self.cfg.get_fluid_blocks())
        self.particle_num = ScalarField(0)

        # ---- allocate the public fields (particle_system.py:89-145) ----
        n = self.particle_max_num
        dev = self.device
        self._t = {}
        for k in _VEC:
            self._t[k] = torch.zeros((n, 3), dtype=torch.float32, device=dev)
        for k in _SCAL_F:
            self._t[k] = torch.zeros(n, dtype=torch.float32, device=dev)
        for k in _SCAL_I:
            self._t[k] = torch.zeros(n, dtype=torch.int32, device=dev)
        self._t["color"] = torch.zeros((n, 3), dtype=torch.int32, device=dev)
        self._t["grid_ids"] = torch.zeros(n, dtype=torch.int32, device=dev)
        self._t["solid_id"] = torch.full((n,), -1, dtype=torch.int32, device=dev)
        C = int(self.grid_num[0] * self.grid_num[1] * self.grid_num[2])
        self._t["grid_particles_num"] = torch.zeros(C, dtype=torch.int32, device=dev)
        if self.simulation_method == 4:  # particle_system.py:115-117
            self._t["dfsph_factor"] = torch.zeros(n, dtype=torch.float32, device=dev)
            self._t["density_adv"] = torch.zeros(n, dtype=torch.float32, device=dev)
            self.dfsph_factor = Field(self, self._t["dfsph_factor"], "dfsph_factor", derived=True)
            self.density_adv = Field(self, self._t["density_adv"], "density_adv", derived=True)
        for k in _PACKED:
            setattr(self, k, Field(self, self._t[k], k))
        self.grid_ids = Field(self, self._t["grid_ids"], "grid_ids", derived=True)
        self.grid_particles_num = Field(self, self._t["grid_particles_num"], "grid_particles_num", derived=True)
        self.grid_particles_num_temp = self.grid_particles_num  # the scan is single-buffer here
        if self.num_rigid_bodies > 0:
            # the reference sizes this num_rigid_bodies + len(fluid_blocks) and indexes it by object id
            # (particle_system.py:91-93); also cover sparse ids
            rows = max(self.num_rigid_bodies + self._n_fluid_blocks, max(self.object_collection) + 1)
            self.rigid_rest_cm = np.full((rows, self.dim), np.nan, np.float32)
        self.x_vis_buffer = None
        if self.GGUI:
            self.x_vis_buffer = torch.zeros((n, 3), dtype=torch.float32, device=dev)
            self.color_vis_buffer = torch.zeros((n, 3), dtype=torch.float32, device=dev)

        # ---- engine ----
        self._dt = self.cfg.get_cfg("timeStepSize") or 1e-4
        # capacity: every solid object could be registered for shape matching
        self._engine = _engine.Engine(self._make_params(), n_max=n, n_solid=self.solid_particle_num + self.emitter_reserve,
                                      n_bodies=self.num_rigid_bodies, device=dev)
        self._fields_dirty = True   # public tensors hold data the engine has not packed yet
        self._engine_ahead = False  # engine state is newer than the public tensors
        self._gpn_stale = True
        self._body_index = {}

        # ---- fill (same order as the reference: fluid blocks, rigid blocks, rigid bodies) ----
        start = 0
        for oid, spec in self.object_collection.items():
            cnt = spec["particleNum"]
            sl = slice(start, start + cnt)
            self.add_particles(oid, cnt, arrays["x"][sl], arrays["v"][sl], arrays["density"][sl],
                               arrays["pressure"][sl], arrays["material"][sl], arrays["is_dynamic"][sl],
                               arrays["color"][sl])
            start += cnt
        self._filled = True

    # ------------------------------------------------------------------------------------
    def _solver_constants(self):
        """The constants the reference bakes into its kernels from the SOLVER's attributes at first launch
        (sph_base.py:13-21, WCSPH.py:9-14): assigning ``solver.viscosity = ...`` etc. takes effect here too
        (at the next engine call; the reference honours it only before its first kernel compile)."""
        cfg, s = self.cfg, getattr(self, "_solver", None)

        def pick(attr, default):
            v = getattr(s, attr, None) if s is not None else None
            return default if v is None else v

        g = pick("g", cfg.get_cfg("gravitation"))
        return (float(pick("density_0", cfg.get_cfg("density0") or 1000.0)),
                float(pick("stiffness", cfg.get_cfg("stiffness") or 50000.0)),
                float(pick("exponent", cfg.get_cfg("exponent") or 7.0)),
                tuple(float(v) for v in np.asarray(g, dtype=np.float64).reshape(-1)),
                float(pick("viscosity", 0.01)), float(pick("surface_tension", 0.01)))

    def _make_params(self, dt=None):
        rho0, stiff, expo, g, visc, sigma = self._solver_constants()
        return _engine.make_params(self.dim, self.grid_num, self.particle_radius, rho0, stiff, expo,
                                   self._dt if dt is None else dt, g, self.domain_size,
                                   viscosity=visc, surface_tension=sigma)

    def _sync_params(self):
        key = (self._dt,) + self._solver_constants()
        if key != getattr(self, "_param_key", None):
            self._engine.set_params(self._make_params())
            self._param_key = key

    def _set_dt(self, dt):
        self._dt = float(dt)
        self._sync_params()

    # ---- field <-> engine coherence -----------------------------------------------------
    def _pull(self, field=None):
        """Make the public tensors current before a read."""
        if field is not None and field.name == "grid_particles_num":
            if self._gpn_stale and not self._fields_dirty:
                self._engine.copy_grid_particles_num(self._t["grid_particles_num"])
                self._gpn_stale = False
            return
        if self._engine_ahead:
            self._engine.unpack(self._t)
            self._engine_ahead = False

    def _touch(self, field=None):
        if field is not None and field._derived:
            raise ValueError(f"{field.name} is produced by the neighbour search and cannot be written")
        self._fields_dirty = True

    def _push(self):
        """Make the engine state current before an engine call."""
        self._sync_params()
        if self._fields_dirty:
            n = int(self.particle_num[None])
            self._prepare_solids(n)
            self._engine.pack(self._t, n, self._n_solid_packed, self._has_dynamic_solids)
            self._fields_dirty = False
            self._gpn_stale = True

    def _after_engine(self):
        self._engine_ahead = True
        self._gpn_stale = True

    def _prepare_solids(self, n):
        """Dense immutable ids for solid particles, each object's solids contiguous."""
        mat = self._t["material"][:n]
        oid = self._t["object_id"][:n]
        solid = (mat == self.material_solid).nonzero(as_tuple=True)[0]
        self._n_solid_packed = int(solid.numel())
        sid = torch.full((self.particle_max_num,), -1, dtype=torch.int32, device=self.device)
        bodies = []
        self._has_dynamic_solids = False
        if self._n_solid_packed:
            order = torch.argsort(oid[solid], stable=True)
            solid_sorted = solid[order]
            sid[solid_sorted] = torch.arange(self._n_solid_packed, dtype=torch.int32, device=self.device)
            self._has_dynamic_solids = bool((self._t["is_dynamic"][:n][solid] != 0).any().item())
            oids_sorted = oid[solid_sorted].cpu().numpy()
            for body_id in sorted(self.object_id_rigid_body):
                if not self.object_collection[body_id]["isDynamic"]:
                    continue
                idx = np.nonzero(oids_sorted == body_id)[0]
                if idx.size:
                    # a re-pack must not forget the rest centre of mass computed at initialize()
                    bodies.append((body_id, int(idx[0]), int(idx[-1]) + 1, self.rigid_rest_cm[body_id]))
        self._t["solid_id"].copy_(sid)
        self._body_index = {b[0]: i for i, b in enumerate(bodies)}
        self._engine.set_rigid_bodies(bodies)

    # ---- reference API --------------------------------------------------------------------
    def build_solver(self):
        solver_type = self.cfg.get_cfg("simulationMethod")
        if solver_type == 0:
            from .WCSPH import WCSPHSolver
            return WCSPHSolver(self)
        if solver_type == 4:
            from .DFSPH import DFSPHSolver
            return DFSPHSolver(self)
        if solver_type == 3:
            from .IISPH import IISPHSolver
            return IISPHSolver(self)
        if solver_type == 1:
            from .PCISPH import PCISPHSolver
            return PCISPHSolver(self)
        raise NotImplementedError(f"Solver type {solver_type} has not been implemented.")

    def add_particles(self, object_id, new_particles_num, new_particles_positions, new_particles_velocity,
                      new_particle_density, new_particle_pressure, new_particles_material,
                      new_particles_is_dynamic, new_particles_color):
        """Append particles (particle_system.py:224-284): x_0 = x, m_V = m_V0, m = m_V0 * density."""
        self._pull()
        p0 = int(self.particle_num[None])
        k = int(new_particles_num)
        if p0 + k > self.particle_max_num:
            raise ValueError(f"add_particles: {p0} + {k} particles exceed particle_max_num = {self.particle_max_num} "
                             "(reserve room with the Configuration key emitterReserve)")
        col = np.asarray(new_particles_color)
        if col.size and (col.min() < 0 or col.max() > 255):
            raise ValueError("colour components must be in 0..255")
        dev = self.device
        sl = slice(p0, p0 + k)

        def up(a, dt):
            return torch.from_numpy(np.ascontiguousarray(np.asarray(a), dtype=dt)).to(dev)

        pos = up(new_particles_positions, np.float32).reshape(k, 3)
        dens = up(new_particle_density, np.float32).reshape(k)
        t = self._t
        t["object_id"][sl] = int(object_id)
        t["x"][sl] = pos
        t["x_0"][sl] = pos
        t["v"][sl] = up(new_particles_velocity, np.float32).reshape(k, 3)
        t["density"][sl] = dens
        t["m_V"][sl] = float(np.float32(self.m_V0))
        t["m"][sl] = dens * float(np.float32(self.m_V0))
        t["pressure"][sl] = up(new_particle_pressure, np.float32).reshape(k)
        t["material"][sl] = up(new_particles_material, np.int32).reshape(k)
        t["is_dynamic"][sl] = up(new_particles_is_dynamic, np.int32).reshape(k)
        t["color"][sl] = up(col, np.int32).reshape(k, 3)
        self.particle_num[None] = p0 + k
        if getattr(self, "_filled", False):  # emitter: particles added after construction
            mat = np.asarray(new_particles_material).reshape(-1)
            self.fluid_particle_num += int((mat == self.material_fluid).sum())
            self.solid_particle_num += int((mat == self.material_solid).sum())
        self._touch()

    def initialize_particle_system(self):
        """update_grid_id + prefix sum + counting_sort (particle_system.py:372-375)."""
        self._push()
        self._engine.neighbor_build()
        self._after_engine()

    # the three phases are one fused neighbour build on the device; the individual names are
    # kept for callers that invoke them in the reference's fixed order.
    def update_grid_id(self):
        self.initialize_particle_system()

    def counting_sort(self):
        pass

    def copy_to_vis_buffer(self, invisible_objects=[]):
        assert self.GGUI
        self._pull()
        if len(invisible_objects) != 0:
            self.x_vis_buffer.fill_(0.0)
            self.color_vis_buffer.fill_(0.0)
        oid = self._t["object_id"]
        for obj_id in self.object_collection:
            if obj_id not in invisible_objects:
                m = oid == obj_id
                self.x_vis_buffer[m] = self._t["x"][m]
                self.color_vis_buffer[m] = self._t["color"][m].to(torch.float32) / 255.0

    def dump(self, obj_id):
        """Positions / velocities of one object in the current sorted order (particle_system.py:409-418)."""
        self._push()
        n = int(self.particle_num[None])
        if n == 0:
            return {"position": np.zeros((0, 3), np.float32), "velocity": np.zeros((0, 3), np.float32)}
        x = torch.empty((n, 3), dtype=torch.float32, device=self.device)
        v = torch.empty((n, 3), dtype=torch.float32, device=self.device)
        oid = torch.empty(n, dtype=torch.int32, device=self.device)
        self._engine.unpack_xv(x, v, oid)
        self._engine.check_status()
        mask = (oid.cpu().numpy() == obj_id).nonzero()
        return {"position": x.cpu().numpy()[mask], "velocity": v.cpu().numpy()[mask]}

    def load_rigid_body(self, rigid_body):
        """Voxelised points of a RigidBodies entry (particle_system.py:421-447)."""
        lattice, verts, faces = rigid_body_lattice(rigid_body, self.particle_diameter, self.cfg.scene_dir)
        if verts is not None:
            rigid_body["restPosition"] = verts
            from .voxelizer import vertex_mean
            rigid_body["restCenterOfMass"] = vertex_mean(verts, rigid_body.get("_vertexWeights"))
            rigid_body["meshFaces"] = faces
        return lattice.astype(np.float64) * self.particle_diameter

    def compute_cube_particle_num(self, start, end):
        return cube_particle_count(start, end, self.particle_diameter)

    def add_cube(self, object_id, lower_corner, cube_size, material, is_dynamic, color=(0, 0, 0), density=None,
                 pressure=None, velocity=None):
        """Lattice block (particle_system.py:458-495)."""
        pos = cube_positions(np.asarray(lower_corner, dtype=np.float64), np.asarray(cube_size, dtype=np.float64),
                             self.particle_diameter)
        k = pos.shape[0]
        vel = np.zeros_like(pos) if velocity is None else np.tile(np.asarray(velocity, np.float32), (k, 1))
        self.add_particles(object_id, k, pos, vel, np.full(k, 1000.0 if density is None else density, np.float32),
                           np.full(k, 0.0 if pressure is None else pressure, np.float32),
                           np.full(k, material, np.int32), np.full(k, int(is_dynamic), np.int32),
                           np.tile(np.asarray(color, np.int32), (k, 1)))

    # ---- host <-> device state exchange (pinned host buffers; used by bench.py's e2e leg) -----
    def _staging(self):
        if getattr(self, "_stage", None) is None:
            n = self.particle_max_num
            self._stage = (torch.empty((n, 3), dtype=torch.float32, device=self.device),
                           torch.empty((n, 3), dtype=torch.float32, device=self.device))
        return self._stage

    def upload_state(self, x_host, v_host):
        """Overwrite positions and velocities (current particle order) from host tensors."""
        self._push()
        sx, sv = self._staging()
        sx.copy_(x_host, non_blocking=True)
        sv.copy_(v_host, non_blocking=True)
        self._engine.upload_xv(sx, sv)
        self._after_engine()

    def download_state(self, x_host, v_host):
        """Copy positions and velocities (current particle order) into host tensors (async)."""
        self._push()
        sx, sv = self._staging()
        self._engine.unpack_xv(sx, sv)
        x_host.copy_(sx, non_blocking=True)
        v_host.copy_(sv, non_blocking=True)
