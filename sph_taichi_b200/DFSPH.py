"""``DFSPHSolver`` (reference ``DFSPH.py:5-408``, simulationMethod 4): divergence-free SPH.

Same method names and constants as the reference; every kernel is one ``sph_dfsph_op`` call on the CUDA engine
(``csrc/sph_dfsph.cuh``).  The density pass builds the per-step neighbour lists that all DFSPH kernels walk.

Two ways to run it, same sweeps, same iteration counts, bit-identical state (``tests/test_gpu_dfsph.py`` runs both
against the oracle):

* ``device_side_loops = True`` (default): ``step()`` is ONE library call (``sph_dfsph_step``) that launches the
  ~50 kernels of a step back to back and runs the two Jacobi loops with the loop condition evaluated on the device
  after every sweep -- one host wait per batch of sweeps, the first batch sized by the previous step's count.
  ``divergence_solve()`` / ``pressure_solve()`` called on their own use ``sph_dfsph_solve`` for the loop.
* ``False`` (or ``SPH_DFSPH_HOST_LOOPS=1``): the reference's structure -- every method below is one launch and the
  loops run on the host (``divergence_solver_iteration`` / ``pressure_solve_iteration``: one density-error read-back
  per sweep).
"""
from __future__ import annotations

import os

import torch

from .sph_base import SPHBase

(OP_DENSITIES, OP_FACTOR, OP_DENSITY_CHANGE, OP_DENSITY_ADV, OP_DENSITY_ERROR, OP_MULTIPLY_FACTOR,
 OP_DIVERGENCE_ITERATION, OP_PRESSURE_ITERATION, OP_NON_PRESSURE, OP_PREDICT_VELOCITY, OP_ADVECT) = range(11)

# The reference solver's constants (DFSPH.py:10-17).  The sharded engine (slab.ShardedSimulation) steps with the same
# ones through dfsph_step_io, so that it matches the single engine it is compared with.
MAX_ITERATIONS_V = MAX_ITERATIONS = 100
MAX_ERROR_V, MAX_ERROR = 0.1, 0.05
FIRST_BATCHES = (2, 3)  # first batch of sweeps of the divergence / pressure solve before a step has counted them


def dfsph_step_io(dt, density0, n_fluid, first_batch_v=FIRST_BATCHES[0], first_batch=FIRST_BATCHES[1], *,
                  enable_divergence_solver=True, max_iterations_v=MAX_ITERATIONS_V, max_iterations=MAX_ITERATIONS,
                  max_error_v=MAX_ERROR_V, max_error=MAX_ERROR):
    """The ``SphDfsphStep`` of ``sph_dfsph_step`` / ``sph_shard_dfsph_step``: the loops' limits and thresholds (eta_v,
    eta as in divergence_solve / pressure_solve) and the multiply_time_step factors of a step of size ``dt``."""
    from ._lib import SphDfsphStep
    return SphDfsphStep(enable_divergence_solver=int(bool(enable_divergence_solver)),
                        max_iterations_v=int(max_iterations_v), max_iterations=int(max_iterations),
                        eta_v=1.0 / dt * max_error_v * 0.01 * density0, eta=max_error * 0.01 * density0,
                        inv_dt=1 / dt, dt=dt, inv_dt2=1 / (dt * dt), density0=density0, n_fluid=int(n_fluid),
                        first_batch_v=first_batch_v, first_batch=first_batch)


class DFSPHSolver(SPHBase):
    _ENGINE_OP, _ENGINE_STEP = "dfsph_op", "dfsph_step"

    def __init__(self, particle_system):
        super().__init__(particle_system)
        self.surface_tension = 0.01
        self.dt[None] = self.ps.cfg.get_cfg("timeStepSize")
        self.enable_divergence_solver = True
        self.m_max_iterations_v = MAX_ITERATIONS_V
        self.m_max_iterations = MAX_ITERATIONS
        self.m_eps = 1e-5
        self.max_error_V = MAX_ERROR_V
        self.max_error = MAX_ERROR
        self.verbose = False
        self.device_side_loops = os.environ.get("SPH_DFSPH_HOST_LOOPS", "0") in ("", "0")  # A/B switch
        self.last_iterations_v = 0
        self.last_iterations = 0
        self._sweeps_guess = list(FIRST_BATCHES)  # first batches of the next two solves (updated every step)
        self.ps._engine.set_dfsph(True)
        self._err = torch.zeros(1, dtype=torch.float64, device=self.ps.device)

    # ---- kernels (DFSPH.py names) ------------------------------------------------------------
    def compute_densities(self):
        self._op(OP_DENSITIES)

    def compute_DFSPH_factor(self):
        self._op(OP_FACTOR)

    def compute_density_change(self):
        self._op(OP_DENSITY_CHANGE)

    def compute_density_adv(self):
        self._op(OP_DENSITY_ADV)

    def compute_density_error(self, offset):
        self._err.zero_()
        self._op(OP_DENSITY_ERROR, offset, self._err)
        return float(self._err.item())  # host sync, like the reference's kernel return value

    def multiply_time_step(self, field, time_step):
        if field is not self.ps.dfsph_factor:
            raise NotImplementedError("the reference only ever scales dfsph_factor")
        self._op(OP_MULTIPLY_FACTOR, time_step)

    def divergence_solver_iteration_kernel(self):
        self._op(OP_DIVERGENCE_ITERATION)

    def pressure_solve_iteration_kernel(self):
        self._op(OP_PRESSURE_ITERATION)

    def compute_non_pressure_forces(self):
        self._op(OP_NON_PRESSURE)

    def predict_velocity(self):
        self._op(OP_PREDICT_VELOCITY)

    def advect(self):
        self._op(OP_ADVECT)

    def _solve_on_device(self, mode, max_iterations, eta, offset):
        self.ps._push()
        it, sweeps, avg = self.ps._engine.dfsph_solve(mode, max_iterations, eta, offset, self.ps.fluid_particle_num,
                                                      self._sweeps_guess[mode])
        self.ps._after_engine()
        self._sweeps_guess[mode] = max(1, sweeps)
        return it, avg

    # ---- convergence loops (DFSPH.py:236-276, 314-352) ----------------------------------------
    def divergence_solver_iteration(self):
        self.divergence_solver_iteration_kernel()
        self.compute_density_change()
        density_err = self.compute_density_error(0.0)
        return density_err / self.ps.fluid_particle_num

    def divergence_solve(self):
        self.compute_density_change()
        inv_dt = 1 / self.dt[None]
        self.multiply_time_step(self.ps.dfsph_factor, inv_dt)
        m_iterations_v = 0
        avg_density_err = 0.0
        if self.device_side_loops:
            eta = 1.0 / self.dt[None] * self.max_error_V * 0.01 * self.density_0
            m_iterations_v, avg_density_err = self._solve_on_device(0, self.m_max_iterations_v, eta, 0.0)
        else:
            while m_iterations_v < 1 or m_iterations_v < self.m_max_iterations_v:
                avg_density_err = self.divergence_solver_iteration()
                eta = 1.0 / self.dt[None] * self.max_error_V * 0.01 * self.density_0
                if avg_density_err <= eta:
                    break
                m_iterations_v += 1
        if self.verbose:
            print(f"DFSPH - iteration V: {m_iterations_v} Avg density err: {avg_density_err}")
        self.multiply_time_step(self.ps.dfsph_factor, self.dt[None])
        self.last_iterations_v = m_iterations_v

    def pressure_solve_iteration(self):
        self.pressure_solve_iteration_kernel()
        self.compute_density_adv()
        density_err = self.compute_density_error(self.density_0)
        return density_err / self.ps.fluid_particle_num

    def pressure_solve(self):
        inv_dt2 = 1 / (self.dt[None] * self.dt[None])
        self.compute_density_adv()
        self.multiply_time_step(self.ps.dfsph_factor, inv_dt2)
        m_iterations = 0
        avg_density_err = 0.0
        if self.device_side_loops:
            eta = self.max_error * 0.01 * self.density_0
            m_iterations, avg_density_err = self._solve_on_device(1, self.m_max_iterations, eta, self.density_0)
        else:
            while m_iterations < 1 or m_iterations < self.m_max_iterations:
                avg_density_err = self.pressure_solve_iteration()
                eta = self.max_error * 0.01 * self.density_0
                if avg_density_err <= eta:
                    break
                m_iterations += 1
        if self.verbose:
            print(f"DFSPH - iterations: {m_iterations} Avg density Err: {avg_density_err:.4f}")
        self.last_iterations = m_iterations

    def step(self, n=1):
        """sph_base.py:263-271.  With device-side loops the whole step is one library call."""
        if not self.device_side_loops:
            return super().step(n)
        io = self._solver_step(n, dfsph_step_io(
            self.dt[None], self.density_0, self.ps.fluid_particle_num, *self._sweeps_guess,
            enable_divergence_solver=self.enable_divergence_solver, max_iterations_v=self.m_max_iterations_v,
            max_iterations=self.m_max_iterations, max_error_v=self.max_error_V, max_error=self.max_error))
        self.last_iterations_v, self.last_iterations = int(io.iterations_v), int(io.iterations)
        if self.verbose:
            print(f"DFSPH - iteration V: {self.last_iterations_v} Avg density err: {io.avg_err_v}")
            print(f"DFSPH - iterations: {self.last_iterations} Avg density Err: {io.avg_err:.4f}")

    def substep(self):
        self.compute_densities()
        self.compute_DFSPH_factor()
        if self.enable_divergence_solver:
            self.divergence_solve()
        self.compute_non_pressure_forces()
        self.predict_velocity()
        self.pressure_solve()
        self.advect()
