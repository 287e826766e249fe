"""``PCISPHSolver`` (simulationMethod 1): predictive-corrective incompressible SPH (Solenthaler & Pajarola 2009).

The reference ships PCISPH only in its legacy 2-D engine (``engine/sph_solver.py``, the ``pci_*`` methods).  This
solver keeps that structure, its method names and its constants (stop once the max density error < 1 % rho0 after at
least 3 iterations, at most 1000 iterations, the pressure reset to 0 every step) and implements the 3-D formulation of
DESIGN.md section 11, which also lists every deviation from the legacy code.  Each method is one ``sph_pcisph_op``
call on the CUDA engine (``csrc/sph_pcisph.cuh``), except ``pci_scaling_factor``, which evaluates delta once on the
host in fp64.

* ``device_side_loops = True`` (default): ``step()`` is ONE library call (``sph_pcisph_step``); the
  prediction-correction loop runs with its condition evaluated on the device after every sweep, one host wait per batch
  of sweeps, the first batch sized by the previous step's count.  ``pressure_solve()`` on its own uses
  ``sph_pcisph_solve``.
* ``False``: the legacy structure -- every method is one op and the loop runs on the host (``pci_pc_iteration``: one
  error read-back per sweep).  Same sweeps, same counts, bit-identical state.
"""
from __future__ import annotations

import numpy as np
import torch

from .fields import ScratchField
from .sph_base import SPHBase

(OP_DENSITIES, OP_COMPUTE_DELTAS, OP_POS_VEL_PREDICTION, OP_UPDATE_PRESSURE, OP_UPDATE_PRESSURE_FORCE,
 OP_PRESSURE_FORCES, OP_UPDATE_TIME_STEP) = range(7)

# the legacy engine's constants
MAX_ERROR = 0.01        # the loop may stop once the max density error < 1 % rho0 ...
MIN_ITERATIONS = 3      # ... and at least this many iterations have run (sub_max_iteration)
MAX_ITERATIONS = 1000
FIRST_BATCH = 4  # first batch of sweeps before a step has counted them


def scaling_factor(dt, particle_radius):
    """pci_scaling_factor in fp64: delta = 1 / (beta (|sum_k gradW_k|^2 + sum_k |gradW_k|^2)), beta = 2 (dt m_V0)^2,
    over the nodes x_k != 0 of the cubic lattice of spacing 2 r (the fluid blocks' lattice) with |x_k| < h = 4 r."""
    d = 2.0 * float(particle_radius)
    h = 4.0 * float(particle_radius)
    m_V0 = 0.8 * d ** 3
    k_dw = 6.0 * 8.0 / np.pi / h ** 3
    n = int(np.ceil(h / d))
    a = np.arange(-n, n + 1, dtype=np.float64)
    x = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3) * d
    r = np.sqrt((x * x).sum(1))
    x, r = x[(r > 0) & (r < h)], r[(r > 0) & (r < h)]
    q = r / h
    f = np.where(q <= 0.5, k_dw * q * (3.0 * q - 2.0), -k_dw * (1.0 - q) ** 2)
    g = (f / (r * h))[:, None] * x
    gs = g.sum(0)
    beta = 2.0 * (float(dt) * m_V0) ** 2
    return 1.0 / (beta * (float(gs @ gs) + float((g * g).sum())))


def pcisph_step_io(delta, first_batch=FIRST_BATCH, *, max_error=MAX_ERROR, min_iterations=MIN_ITERATIONS,
                   max_iterations=MAX_ITERATIONS):
    """The ``SphPcisphStep`` of ``sph_pcisph_step``: delta (rounded to fp32), the loop's threshold (eta: a fraction of
    rho0), its minimum and maximum iteration counts and the first batch of sweeps."""
    from ._lib import SphPcisphStep
    return SphPcisphStep(delta=float(np.float32(delta)), eta=float(max_error), min_iterations=int(min_iterations),
                         max_iterations=int(max_iterations), first_batch=int(first_batch))


class PCISPHSolver(SPHBase):
    _ENGINE_OP, _ENGINE_STEP = "pcisph_op", "pcisph_step"

    def __init__(self, particle_system):
        super().__init__(particle_system)
        self.surface_tension = 0.0  # the non-pressure forces are gravity + viscosity
        self.dt[None] = self.ps.cfg.get_cfg("timeStepSize")
        self.max_error = MAX_ERROR
        self.sub_max_iteration = MIN_ITERATIONS
        self.max_iterations = MAX_ITERATIONS
        self.verbose = False
        self.device_side_loops = True
        self.s_f = 0.0  # delta, the legacy engine's name
        self.last_iterations = 0
        self.last_max_density_error = 0.0
        self._sweeps_guess = FIRST_BATCH
        self.ps._engine.set_pcisph(True)
        self._err = torch.zeros(1, dtype=torch.int32, device=self.ps.device)
        self.predicted_density = ScratchField(self, "pcisph_read", 0, 1)
        self.pressure_accel = ScratchField(self, "pcisph_read", 2, 3)
        self.pci_scaling_factor()

    def step_io(self):
        """The ``SphPcisphStep`` of ``sph_pcisph_step`` from this solver's constants."""
        return pcisph_step_io(self.s_f, self._sweeps_guess, max_error=self.max_error,
                              min_iterations=self.sub_max_iteration, max_iterations=self.max_iterations)

    def _done(self, err, it):
        rho0 = self.ps._solver_constants()[0]  # the engine's rho0
        return (err < self.max_error * rho0 and it >= self.sub_max_iteration) or it >= self.max_iterations

    # ---- kernels (the legacy engine's names) -----------------------------------------------------
    def compute_densities(self):
        self._op(OP_DENSITIES)

    def pci_compute_deltas(self):
        self._op(OP_COMPUTE_DELTAS)

    def pci_scaling_factor(self):
        """delta once per time step size, in fp64 on the host (the legacy code recomputes it every step)."""
        self.s_f = scaling_factor(self.dt[None], self.ps.particle_radius)
        return self.s_f

    def pci_pos_vel_prediction(self):
        self._op(OP_POS_VEL_PREDICTION)

    def pci_update_pressure(self):
        """Predicted density, pressure update and the sweep's max error; returns the error (host sync, like the
        legacy field read)."""
        self._err.zero_()
        self._op(OP_UPDATE_PRESSURE, float(np.float32(self.s_f)), self._err)
        return float(self._err.cpu().view(torch.float32).item())

    def pci_update_pressure_force(self):
        self._op(OP_UPDATE_PRESSURE_FORCE)

    def pci_pc_iteration(self):
        self.pci_pos_vel_prediction()
        err = self.pci_update_pressure()
        self.pci_update_pressure_force()
        return err

    def pressure_solve(self):
        """The prediction-correction loop (after pci_compute_deltas)."""
        self.pci_scaling_factor()
        if self.device_side_loops:
            self.ps._push()
            it, err = self.ps._engine.pcisph_solve(float(np.float32(self.s_f)), self.max_error, self.sub_max_iteration,
                                                    self.max_iterations, self._sweeps_guess)
            self.ps._after_engine()
            self._sweeps_guess = max(1, it)
        else:
            it, err = 0, 0.0
            while True:
                err = self.pci_pc_iteration()
                it += 1
                if self._done(err, it):
                    break
        if self.verbose:
            print(f"PCISPH - iterations: {it} Max density err: {err:.3e}")
        self.last_iterations, self.last_max_density_error = it, err

    def compute_pressure_forces(self):
        self._op(OP_PRESSURE_FORCES)

    def pci_update_time_step(self):
        self._op(OP_UPDATE_TIME_STEP)

    def substep(self):
        self.compute_densities()
        self.pci_compute_deltas()
        self.pressure_solve()
        self.compute_pressure_forces()
        self.pci_update_time_step()

    def step(self, n=1):
        """sph_base.py:263-271.  With device-side loops the whole step is one library call."""
        if not self.device_side_loops:
            return super().step(n)
        self.pci_scaling_factor()
        io = self._solver_step(n, self.step_io())
        self.last_iterations, self.last_max_density_error = int(io.iterations), float(io.max_err)
        if self.verbose:
            print(f"PCISPH - iterations: {self.last_iterations} Max density err: {self.last_max_density_error:.3e}")
