"""``IISPHSolver`` (reference ``IISPH.py``, simulationMethod 3): implicit incompressible SPH (Ihmsen et al. 2014).

The reference's ``IISPH.py`` cannot run (its ``build_solver`` never constructs it, it reads neighbour fields its
``ParticleSystem`` no longer has, and its kernels have indexing errors).  This solver keeps its method names, its
structure and its constants (omega = 0.5, warm start with 0.5 p, stop when the average error < 1e-3, at most 1000
sweeps, Akinci boundary with mirrored pressure) and implements the formulation of DESIGN.md section 10, which also
lists every deviation from ``IISPH.py``.  Each method is one ``sph_iisph_op`` call on the CUDA engine
(``csrc/sph_iisph.cuh``).

* ``device_side_loops = True`` (default): ``step()`` is ONE library call (``sph_iisph_step``); the Jacobi loop runs
  with its condition evaluated on the device after every sweep, one host wait per batch of sweeps, the first batch
  sized by the previous step's count.  ``pressure_solve()`` called on its own uses ``sph_iisph_solve``.
* ``False``: the reference's structure -- every method is one op and the loop runs on the host
  (``pressure_solve_iteration``: one error read-back per sweep).  Same sweeps, same counts, bit-identical state.
"""
from __future__ import annotations

import torch

from .sph_base import SPHBase

(OP_DENSITIES, OP_NON_PRESSURE, OP_PREDICT_ADVECTION, OP_PRESSURE_SOLVE_ITERATION, OP_PRESSURE_FORCES,
 OP_ADVECT) = range(6)

# IISPH.py's constants
OMEGA = 0.5
MAX_ITERATIONS = 1000
MAX_ERROR = 1e-3
FIRST_BATCH = 4  # first batch of sweeps before a step has counted them


def iisph_step_io(n_fluid, first_batch=FIRST_BATCH, *, omega=OMEGA, max_iterations=MAX_ITERATIONS,
                  max_error=MAX_ERROR):
    """The ``SphIisphStep`` of ``sph_iisph_step`` / ``sph_shard_iisph_step``: the loop's limit, relaxation and threshold
    (eta = the average error below which pressure_solve stops), the fluid count the error is averaged over (sharded:
    the fluid particles of ALL ranks) and the first batch of sweeps."""
    from ._lib import SphIisphStep
    return SphIisphStep(max_iterations=int(max_iterations), omega=float(omega), eta=float(max_error),
                        n_fluid=int(n_fluid), first_batch=int(first_batch))


class _ScratchField:
    """Read-only per-particle scratch of the last IISPH kernels (a_ii, s_i or a^p), in the public fields' order."""

    def __init__(self, solver, which, width):
        self._solver, self._which, self._width = solver, which, width

    @property
    def shape(self):
        return (self._solver.ps.particle_max_num,)

    def to_numpy(self):
        ps = self._solver.ps
        ps._push()
        n = ps.particle_max_num
        out = torch.zeros((n, 3) if self._width == 3 else (n,), dtype=torch.float32, device=ps.device)
        args = [None, None, None]
        args[self._which] = out
        ps._engine.iisph_read(*args)
        return out.cpu().numpy()


class IISPHSolver(SPHBase):
    def __init__(self, particle_system):
        super().__init__(particle_system)
        self.surface_tension = 0.0  # IISPH.py's non-pressure forces are gravity + viscosity
        self.dt[None] = self.ps.cfg.get_cfg("timeStepSize")
        self.omega = OMEGA
        self.max_iterations = MAX_ITERATIONS
        self.max_error = MAX_ERROR
        self.verbose = False
        self.device_side_loops = True
        self.last_iterations = 0
        self.last_avg_density_error = 0.0
        self._sweeps_guess = FIRST_BATCH
        self.ps._engine.set_iisph(True)
        self._err = torch.zeros(1, dtype=torch.float64, device=self.ps.device)
        self.a_ii = _ScratchField(self, 0, 1)
        self.density_deviation = _ScratchField(self, 1, 1)
        self.pressure_accel = _ScratchField(self, 2, 3)

    def _op(self, op, arg=0.0, out=None):
        self.ps._push()
        self.ps._engine.iisph_op(op, arg, out)
        self.ps._after_engine()

    def step_io(self):
        """The ``SphIisphStep`` of ``sph_iisph_step`` from this solver's constants."""
        return iisph_step_io(self.ps.fluid_particle_num, self._sweeps_guess, omega=self.omega,
                             max_iterations=self.max_iterations, max_error=self.max_error)

    # ---- kernels (IISPH.py names) ------------------------------------------------------------
    def compute_densities(self):
        self._op(OP_DENSITIES)

    def compute_non_pressure_forces(self):
        self._op(OP_NON_PRESSURE)

    def predict_advection(self):
        self._op(OP_PREDICT_ADVECTION)

    def pressure_solve_iteration(self):
        """One relaxed Jacobi sweep; returns the average error (host sync, like the reference's field read)."""
        self._err.zero_()
        self._op(OP_PRESSURE_SOLVE_ITERATION, self.omega, self._err)
        return float(self._err.item()) / self.ps.fluid_particle_num

    def pressure_solve(self):
        if self.device_side_loops:
            self.ps._push()
            it, avg = self.ps._engine.iisph_solve(self.max_iterations, self.omega, self.max_error,
                                                   self.ps.fluid_particle_num, self._sweeps_guess)
            self.ps._after_engine()
            self._sweeps_guess = max(1, it)
        else:
            it, avg = 0, 0.0
            while it < self.max_iterations:
                avg = self.pressure_solve_iteration()
                it += 1
                if avg < self.max_error:
                    break
        if self.verbose:
            print(f"IISPH - iterations: {it} Avg density err: {avg:.3e}")
        self.last_iterations, self.last_avg_density_error = it, avg

    def compute_pressure_forces(self):
        self._op(OP_PRESSURE_FORCES)

    def advect(self):
        self._op(OP_ADVECT)

    def substep(self):
        self.compute_densities()
        self.compute_non_pressure_forces()
        self.predict_advection()
        self.pressure_solve()
        self.compute_pressure_forces()
        self.advect()

    def step(self, n=1):
        """sph_base.py:263-271.  With device-side loops the whole step is one library call."""
        if not self.device_side_loops:
            return super().step(n)
        ps = self.ps
        io = self.step_io()
        ps._push()
        ps._engine.iisph_step(n, io)
        ps._after_engine()
        self._sweeps_guess = int(io.first_batch)
        self.last_iterations, self.last_avg_density_error = int(io.iterations), float(io.avg_err)
        if self.verbose:
            print(f"IISPH - iterations: {self.last_iterations} Avg density err: {self.last_avg_density_error:.3e}")
        if ps.cfg.get_cfg("exportObj"):
            for oid in ps._body_index:
                if "restPosition" in ps.object_collection[oid]:
                    self._update_mesh(oid)
