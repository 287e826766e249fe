"""Thin object wrapper over the C ABI: owns the torch workspace and the context handle.

PyTorch is used for device memory and streams only; every device computation is a kernel of
``libsph_b200.so``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

STATUS_OUT_OF_GRID = 1
STATUS_BAD_POLAR = 2


def make_params(dim, grid_num, particle_radius, density0, stiffness, exponent, dt, gravitation, domain_size,
                viscosity=0.01, surface_tension=0.01):
    """Fold all constants in double exactly where the reference folds them in Python scope."""
    d = 2 * particle_radius
    h = particle_radius * 4.0
    k = 8 / np.pi / h ** dim  # sph_base.py:27-35 (3-D)
    p = _lib.SphParams()
    p.dim = dim
    p.grid_num = (C.c_int32 * 3)(*[int(v) for v in grid_num])
    p.h = h
    p.diameter = d
    p.m_V0 = 0.8 * d ** dim
    p.density0 = density0
    p.stiffness = stiffness
    p.exponent = exponent
    p.viscosity = viscosity
    p.surface_tension = surface_tension
    p.dt = dt
    p.g = (C.c_float * 3)(*[float(v) for v in gravitation])
    p.domain_size = (C.c_float * 3)(*[float(v) for v in domain_size])
    p.k_w = k
    p.k_dw = 6.0 * k
    p.visc_eps = 0.01 * h ** 2
    p.clamp_hi = (C.c_float * 3)(*[float(v) - h for v in domain_size])
    return p


class Engine:
    def __init__(self, params, n_max, n_solid=0, n_bodies=0, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("sph_taichi_b200 needs a CUDA device: the engine is hand-written sm_90a CUDA "
                               "with no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.params = params
        self.n_max = int(n_max)
        self.n_solid_cap = int(n_solid)
        nbytes = self.lib.sph_workspace_bytes(C.byref(params), self.n_max, self.n_solid_cap, int(n_bodies))
        if nbytes == 0:
            raise ValueError("invalid SPH parameters (grid must be >= 3 cells per axis, dim == 3)")
        with torch.cuda.device(self.device):
            self.workspace = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
        base = self.workspace.data_ptr()
        self._ws_ptr = (base + 255) // 256 * 256
        handle = C.c_void_p()
        rc = self.lib.sph_create(C.byref(params), self.n_max, self.n_solid_cap, int(n_bodies), self.device.index or 0,
                                 C.c_void_p(self._ws_ptr), int(nbytes), C.byref(handle))
        if rc:
            raise RuntimeError(f"sph_create failed ({rc}): {self.lib.sph_last_error(None).decode()}")
        self.ctx = handle

    # -- helpers ----------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check(self, rc, what):
        if rc < 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.sph_last_error(self.ctx).decode()}")
        return rc

    def close(self):
        if getattr(self, "ctx", None):
            torch.cuda.synchronize(self.device)
            self.lib.sph_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def fields_struct(tensors):
        f = _lib.SphFields()
        for k, _ in _lib.SphFields._fields_:
            t = tensors.get(k)
            setattr(f, k, None if t is None else t.data_ptr())
        return f

    # -- ABI ------------------------------------------------------------------------------
    def set_params(self, params):
        self.params = params
        self._check(self.lib.sph_set_params(self.ctx, C.byref(params)), "sph_set_params")

    def pack(self, tensors, n, n_solid, has_dynamic_solids, uniform_hint=None):
        """uniform_hint = (uniform, fluid_m, fluid_mV) decided by the caller for the WHOLE scene (sharded runs: a
        rank that starts without particles must still run the same kernels as its peers); None derives it here."""
        self._check(self.lib.sph_set_solid_count(self.ctx, int(n_solid), int(bool(has_dynamic_solids))),
                    "sph_set_solid_count")
        # uniform-fluid hint: all fluid particles share one m and one m_V (bitwise)
        uniform, fm, fmv = 0, 0.0, 0.0
        if uniform_hint is not None:
            uniform, fm, fmv = int(bool(uniform_hint[0])), float(uniform_hint[1]), float(uniform_hint[2])
        elif n > 0:
            fluid = tensors["material"][:n] == 1
            if bool(fluid.any().item()):
                m, mv = tensors["m"][:n][fluid], tensors["m_V"][:n][fluid]
                fm, fmv = float(m[0].item()), float(mv[0].item())
                uniform = int(bool((m == m[0]).all().item()) and bool((mv == mv[0]).all().item()))
        self._check(self.lib.sph_set_fluid_uniform(self.ctx, uniform, fm, fmv), "sph_set_fluid_uniform")
        f = self.fields_struct(tensors)
        self._check(self.lib.sph_pack(self.ctx, C.byref(f), int(n), self._stream()), "sph_pack")

    def unpack(self, tensors):
        f = self.fields_struct(tensors)
        self._check(self.lib.sph_unpack(self.ctx, C.byref(f), self._stream()), "sph_unpack")

    def unpack_xv(self, x, v, object_id=None):
        self._check(self.lib.sph_unpack_xv(self.ctx, x.data_ptr(), v.data_ptr(),
                                           None if object_id is None else object_id.data_ptr(), self._stream()),
                    "sph_unpack_xv")

    def upload_xv(self, x, v):
        self._check(self.lib.sph_upload_xv(self.ctx, x.data_ptr(), v.data_ptr(), self._stream()), "sph_upload_xv")

    def copy_grid_particles_num(self, out):
        self._check(self.lib.sph_copy_grid_particles_num(self.ctx, out.data_ptr(), self._stream()),
                    "sph_copy_grid_particles_num")

    def neighbor_build(self):
        self._check(self.lib.sph_neighbor_build(self.ctx, self._stream()), "sph_neighbor_build")

    def boundary_volume(self, moving):
        self._check(self.lib.sph_boundary_volume(self.ctx, int(moving), self._stream()), "sph_boundary_volume")

    def compute_densities(self):
        self._check(self.lib.sph_compute_densities(self.ctx, self._stream()), "sph_compute_densities")

    def compute_non_pressure_forces(self):
        self._check(self.lib.sph_compute_non_pressure_forces(self.ctx, self._stream()),
                    "sph_compute_non_pressure_forces")

    def compute_pressure_forces(self):
        self._check(self.lib.sph_compute_pressure_forces(self.ctx, self._stream()), "sph_compute_pressure_forces")

    def advect(self):
        self._check(self.lib.sph_advect(self.ctx, self._stream()), "sph_advect")

    def enforce_boundary(self, particle_type):
        self._check(self.lib.sph_enforce_boundary(self.ctx, int(particle_type), self._stream()),
                    "sph_enforce_boundary")

    def set_rigid_bodies(self, bodies):
        arr = (_lib.SphRigidBody * max(1, len(bodies)))()
        for i, (oid, b0, b1, rest_cm) in enumerate(bodies):
            arr[i].object_id, arr[i].solid_begin, arr[i].solid_end = int(oid), int(b0), int(b1)
            arr[i].rest_cm = (C.c_float * 3)(*[float(v) for v in rest_cm])
        self._check(self.lib.sph_set_rigid_bodies(self.ctx, arr, len(bodies)), "sph_set_rigid_bodies")

    def compute_com(self, body_index):
        out = torch.empty(3, dtype=torch.float32, device=self.device)
        self._check(self.lib.sph_compute_com(self.ctx, int(body_index), out.data_ptr(), self._stream()),
                    "sph_compute_com")
        return out

    def compute_rigid_rest_cm(self, body_index):
        self._check(self.lib.sph_compute_rigid_rest_cm(self.ctx, int(body_index), self._stream()),
                    "sph_compute_rigid_rest_cm")

    def solve_constraints(self, body_index):
        out = torch.empty(9, dtype=torch.float32, device=self.device)
        self._check(self.lib.sph_solve_constraints(self.ctx, int(body_index), out.data_ptr(), self._stream()),
                    "sph_solve_constraints")
        return out.view(3, 3)

    def rigid_state(self, body_index):
        """(R [3,3], cm [3]) of the body's last shape-matching solve, as numpy arrays."""
        out = torch.empty(12, dtype=torch.float32, device=self.device)
        self._check(self.lib.sph_get_rigid_state(self.ctx, int(body_index), out.data_ptr(), self._stream()),
                    "sph_get_rigid_state")
        h = out.cpu().numpy()
        return h[:9].reshape(3, 3), h[9:]

    def set_dfsph(self, enable=True):
        self._check(self.lib.sph_set_dfsph(self.ctx, int(bool(enable))), "sph_set_dfsph")

    def dfsph_op(self, op, arg=0.0, out=None):
        self._check(self.lib.sph_dfsph_op(self.ctx, int(op), float(arg), None if out is None else out.data_ptr(),
                                          self._stream()), "sph_dfsph_op")

    def dfsph_solve(self, mode, max_iterations, eta, offset, n_fluid, first_batch):
        """The Jacobi loop of divergence_solve (mode 0) / pressure_solve (mode 1) with the loop condition on the
        device; returns (iterations, sweeps, last avg_density_err).  Synchronous (one wait per batch of sweeps)."""
        it, sw, avg = C.c_int32(0), C.c_int32(0), C.c_double(0.0)
        self._check(self.lib.sph_dfsph_solve(self.ctx, int(mode), int(max_iterations), float(eta), float(offset),
                                             int(n_fluid), int(first_batch), C.byref(it), C.byref(sw), C.byref(avg),
                                             self._stream()), "sph_dfsph_solve")
        return int(it.value), int(sw.value), float(avg.value)

    def dfsph_step(self, nsteps, io):
        """`nsteps` whole DFSPH steps launched from one call; `io` is a _lib.SphDfsphStep (constants in, counts out)."""
        self._check(self.lib.sph_dfsph_step(self.ctx, int(nsteps), C.byref(io), self._stream()), "sph_dfsph_step")

    def set_iisph(self, enable=True):
        self._check(self.lib.sph_set_iisph(self.ctx, int(bool(enable))), "sph_set_iisph")

    def iisph_op(self, op, arg=0.0, out=None):
        self._check(self.lib.sph_iisph_op(self.ctx, int(op), float(arg), None if out is None else out.data_ptr(),
                                          self._stream()), "sph_iisph_op")

    def iisph_solve(self, max_iterations, omega, eta, n_fluid, first_batch):
        """pressure_solve's Jacobi loop with the loop condition on the device; returns (iterations, last average
        error).  Synchronous (one wait per batch of sweeps)."""
        it, avg = C.c_int32(0), C.c_double(0.0)
        self._check(self.lib.sph_iisph_solve(self.ctx, int(max_iterations), float(omega), float(eta), int(n_fluid),
                                             int(first_batch), C.byref(it), C.byref(avg), self._stream()),
                    "sph_iisph_solve")
        return int(it.value), float(avg.value)

    def iisph_step(self, nsteps, io):
        """`nsteps` whole IISPH steps launched from one call; `io` is a _lib.SphIisphStep (constants in, counts out)."""
        self._check(self.lib.sph_iisph_step(self.ctx, int(nsteps), C.byref(io), self._stream()), "sph_iisph_step")

    def iisph_read(self, a_ii=None, s=None, ap=None):
        """a_ii [n], s [n], a^p [n, 3] (float32 tensors on the engine's device, each may be None), sorted order."""
        ptr = [None if t is None else t.data_ptr() for t in (a_ii, s, ap)]
        self._check(self.lib.sph_iisph_read(self.ctx, *ptr, self._stream()), "sph_iisph_read")

    def set_pcisph(self, enable=True):
        self._check(self.lib.sph_set_pcisph(self.ctx, int(bool(enable))), "sph_set_pcisph")

    def pcisph_op(self, op, arg=0.0, out=None):
        self._check(self.lib.sph_pcisph_op(self.ctx, int(op), float(arg), None if out is None else out.data_ptr(),
                                           self._stream()), "sph_pcisph_op")

    def pcisph_solve(self, delta, eta, min_iterations, max_iterations, first_batch):
        """The prediction-correction loop with its condition on the device; returns (iterations, last max error).
        Synchronous (one wait per batch of sweeps)."""
        it, err = C.c_int32(0), C.c_double(0.0)
        self._check(self.lib.sph_pcisph_solve(self.ctx, float(delta), float(eta), int(min_iterations),
                                              int(max_iterations), int(first_batch), C.byref(it), C.byref(err),
                                              self._stream()), "sph_pcisph_solve")
        return int(it.value), float(err.value)

    def pcisph_step(self, nsteps, io):
        """`nsteps` whole PCISPH steps launched from one call; `io` is a _lib.SphPcisphStep (constants in, counts
        out)."""
        self._check(self.lib.sph_pcisph_step(self.ctx, int(nsteps), C.byref(io), self._stream()), "sph_pcisph_step")

    def pcisph_read(self, rho_star=None, p=None, ap=None):
        """rho* [n], p [n], a^p [n, 3] (float32 tensors on the engine's device, each may be None), sorted order."""
        ptr = [None if t is None else t.data_ptr() for t in (rho_star, p, ap)]
        self._check(self.lib.sph_pcisph_read(self.ctx, *ptr, self._stream()), "sph_pcisph_read")

    def step(self, nsteps=1):
        self._check(self.lib.sph_step(self.ctx, int(nsteps), self._stream()), "sph_step")

    def read_status(self):
        st = C.c_uint32(0)
        self._check(self.lib.sph_read_status(self.ctx, C.byref(st), self._stream()), "sph_read_status")
        return int(st.value)

    def clear_status(self):
        self._check(self.lib.sph_clear_status(self.ctx, self._stream()), "sph_clear_status")

    def check_status(self):
        st = self.read_status()
        if st & STATUS_OUT_OF_GRID:
            raise RuntimeError("a particle left the grid (NaN or outside [0, domain)): the reference would write "
                               "out of bounds here")
        return st

    def neighbor_stats(self):
        """{max, overflow, pairs, fluid} of the neighbour lists built by the last density pass."""
        out = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._check(self.lib.sph_neighbor_stats(self.ctx, out.data_ptr(), self._stream()), "sph_neighbor_stats")
        m, o, p, f = (int(v) for v in out.cpu().tolist())
        return {"max": m, "overflow": o, "pairs": p, "fluid": f, "mean": p / max(f, 1)}

    def launch_count(self):
        return int(self.lib.sph_launch_count(self.ctx))

    def particle_count(self):
        return int(self.lib.sph_particle_count(self.ctx))

    def profile_step(self):
        buf = (C.c_float * 16)()
        n = self._check(self.lib.sph_profile_step(self.ctx, buf, 16, self._stream()), "sph_profile_step")
        return {self.lib.sph_timer_name(i).decode(): float(buf[i]) for i in range(n)}
