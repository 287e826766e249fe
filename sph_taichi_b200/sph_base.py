"""``SPHBase``: step orchestration, boundary volumes, wall clamp and shape-matching rigid bodies
(reference ``sph_base.py:7-271``) as a shell over the CUDA engine.

``step()`` takes the fused, CUDA-graph-replayed path (``sph_step``) whenever ``substep`` is the
stock WCSPH one; a subclass that overrides ``substep`` gets the reference's generic sequence of
individual calls instead (sph_base.py:263-271).
"""
from __future__ import annotations

import numpy as np

from .fields import ScalarField


def posed_mesh(rest, rest_cm, R, cm):
    """Vertices of a rigid body's mesh in its current pose (sph_base.py:253-257): cm + R (rest - rest_cm).  The OBJ
    export of the single engine (``SPHBase._update_mesh``) and of a sharded run (``run_simulation.py --gpus``)."""
    ret = R @ (rest - rest_cm).T
    return cm + ret.T


class SPHBase:
    def __init__(self, particle_system):
        self.ps = particle_system
        self.ps._solver = self  # the engine constants follow this object's attributes (ps._solver_constants)
        self.g = np.array(self.ps.cfg.get_cfg("gravitation"))
        self.viscosity = 0.01      # sph_base.py:15
        self.density_0 = self.ps.cfg.get_cfg("density0")
        self.dt = ScalarField(1e-4, on_change=self.ps._set_dt)  # sph_base.py:20-21
        self._rigid_R = {}

    # ---- initialisation (sph_base.py:80-113) ------------------------------------------------
    def initialize(self):
        self.ps.initialize_particle_system()
        for r_obj_id in sorted(self.ps.object_id_rigid_body):
            self.compute_rigid_rest_cm(r_obj_id)
        self.compute_static_boundary_volume()
        self.compute_moving_boundary_volume()

    def compute_rigid_rest_cm(self, object_id):
        ps = self.ps
        ps._push()
        b = ps._body_index.get(object_id)
        if b is None:
            return  # static body: the reference stores 0/0 = NaN and never reads it (SURVEY Q8)
        ps._engine.compute_rigid_rest_cm(b)
        ps.rigid_rest_cm[object_id] = ps._engine.compute_com(b).cpu().numpy()

    def compute_static_boundary_volume(self):
        self.ps._push()
        self.ps._engine.boundary_volume(0)
        self.ps._after_engine()

    def compute_moving_boundary_volume(self):
        self.ps._push()
        self.ps._engine.boundary_volume(1)
        self.ps._after_engine()

    def substep(self):
        pass

    # ---- walls (sph_base.py:118-179) -----------------------------------------------------------
    def enforce_boundary_3D(self, particle_type):
        self.ps._push()
        self.ps._engine.enforce_boundary(particle_type)
        self.ps._after_engine()

    # ---- rigid bodies (sph_base.py:182-260) ----------------------------------------------------
    def compute_com_kernel(self, object_id):
        ps = self.ps
        ps._push()
        b = ps._body_index.get(object_id)
        if b is None:
            return np.full(3, np.nan, np.float32)
        return ps._engine.compute_com(b).cpu().numpy()

    def solve_constraints(self, object_id):
        """Shape matching of one dynamic body; returns a lazily downloaded 3x3 R."""
        ps = self.ps
        ps._push()
        b = ps._body_index.get(object_id)
        if b is None:
            raise ValueError(f"object {object_id} is not a dynamic rigid body")
        R = ps._engine.solve_constraints(b)
        ps._after_engine()
        self._rigid_R[object_id] = R
        return R

    def solve_rigid_body(self):
        ps = self.ps
        for r_obj_id in sorted(ps.object_id_rigid_body):
            if ps.object_collection[r_obj_id]["isDynamic"]:
                R = self.solve_constraints(r_obj_id)
                if ps.cfg.get_cfg("exportObj") and "restPosition" in ps.object_collection[r_obj_id]:
                    self._update_mesh(r_obj_id, R)
                self.enforce_boundary_3D(ps.material_solid)

    def _update_mesh(self, r_obj_id, R=None):
        """Posed mesh vertices for the OBJ export (sph_base.py:253-257): cm + R (rest - rest_cm)."""
        ps = self.ps
        obj = ps.object_collection[r_obj_id]
        if R is None:  # fused step: R and cm stayed on the device
            R, cm = ps._engine.rigid_state(ps._body_index[r_obj_id])
        else:
            R, cm = R.cpu().numpy(), self.compute_com_kernel(r_obj_id)
        obj["meshVertices"] = posed_mesh(obj["restPosition"], obj["restCenterOfMass"], R, cm)

    # ---- step (sph_base.py:263-271) ----------------------------------------------------------------
    def _fused_step_ok(self):
        return False

    def step(self, n=1):
        ps = self.ps
        if self._fused_step_ok():
            ps._push()
            ps._engine.step(n)
            ps._after_engine()
            if ps.cfg.get_cfg("exportObj"):
                for oid in ps._body_index:
                    if "restPosition" in ps.object_collection[oid]:
                        self._update_mesh(oid)
            return
        for _ in range(n):
            ps.initialize_particle_system()
            self.compute_moving_boundary_volume()
            self.substep()
            self.solve_rigid_body()
            self.enforce_boundary_3D(ps.material_fluid)
