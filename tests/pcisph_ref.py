"""Numpy restatement of the PCISPH formulation of DESIGN.md section 11 (TEST INFRASTRUCTURE ONLY).

Steps 3-7 of a PCISPH step (pci_compute_deltas' resets, the prediction-correction loop, compute_pressure_forces with
the reactions, pci_update_time_step) on the arrays of an ``oracle.sph_oracle.OracleSim`` (fp32 or fp64), which
supplies everything else: the neighbour sort, boundary volumes, the density pass and the non-pressure forces (with
``surface_tension = 0``), shape matching and the wall clamps.  The step's neighbour pairs are found at x^t with a k-d
tree and kept by the reference's exact predicate ``(x_i - x_j).norm() < h`` in the simulation's precision, so the
pair set is the engine's; every sweep then evaluates them at the predicted positions.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from tests.iisph_ref import iisph_oracle

MAX_ERROR, MIN_ITERATIONS, MAX_ITERATIONS = 0.01, 3, 1000


def pcisph_oracle(sc, f64=False):
    """An OracleSim of a PCISPH scene: its density pass and non-pressure forces are DFSPH's without cohesion."""
    return iisph_oracle(sc, f64=f64)


class PcisphRef:
    def __init__(self, o, delta):
        self.o = o
        self.r = o.real
        r = self.r
        self.dt = r(o.P.dt)
        self.rho0 = r(o.P.density0)
        self.h = r(o.support_radius)
        k = 8 / np.pi / float(o.support_radius) ** 3
        self.k_w, self.k_dw = r(k), r(6.0 * k)
        self.delta = r(delta)
        self.last_iterations, self.last_err = 0, 0.0

    # ---- geometry ------------------------------------------------------------------------------------------------
    def pairs(self):
        """(i, j) for every fluid i and neighbour j != i at x^t: the step's lists."""
        o, r = self.o, self.r
        x = o.x.astype(r)
        tree = cKDTree(x.astype(np.float64))
        pr = tree.query_pairs(float(self.h) * (1 + 1e-5), output_type="ndarray")
        i = np.concatenate([pr[:, 0], pr[:, 1]])
        j = np.concatenate([pr[:, 1], pr[:, 0]])
        d = x[i] - x[j]
        rn = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        keep = (rn < self.h) & (o.material[i] == 1)
        self.i, self.j = i[keep], j[keep]
        self.fl_j = o.material[self.j] == 1
        return self.i, self.j

    def _rq(self):
        """r = x*_i - x*_j, |r| and q = |r| / h over the pairs."""
        d = (self.xs[self.i] - self.xs[self.j]).astype(self.r)
        rn = np.sqrt((d * d).sum(1)).astype(self.r)
        return d, rn, (rn / self.h).astype(self.r)

    def W(self, q):
        r = self.r
        f = np.maximum(r(1) - q, r(0))
        return np.where(q <= r(0.5), self.k_w * (r(6) * q ** 3 - r(6) * q * q + r(1)),
                        r(2) * self.k_w * f * f * f).astype(r)

    def gradW(self, d, rn, q):
        r = self.r
        ok = (rn > r(1e-5)) & (q <= r(1))
        f = r(1) - q
        res = np.where(q <= r(0.5), self.k_dw * q * (r(3) * q - r(2)), self.k_dw * (-f * f))
        safe = np.where(ok, rn, r(1))
        return np.where(ok[:, None], (res / (safe * self.h))[:, None] * d, r(0)).astype(r)

    def _sum(self, vals):
        out = np.zeros((self.o.n,) + vals.shape[1:], dtype=vals.dtype)
        np.add.at(out, self.i, vals)
        return out

    # ---- steps 3-7 -----------------------------------------------------------------------------------------------
    def compute_deltas(self):
        """After the oracle's density pass and non-pressure forces: a^np, p = 0, a^p = 0, x* = x."""
        o, r = self.o, self.r
        self.pairs()
        fl = o.material == 1
        self.anp = o.acceleration.astype(r).copy()
        o.pressure[fl] = 0
        self.ap = np.zeros((o.n, 3), r)
        self.xs = o.x.astype(r).copy()
        self.rho_star = np.zeros(o.n, r)

    def _velocity(self):
        o = self.o
        return (o.v + self.dt * (self.anp + self.ap)).astype(self.r)

    def predict(self):
        o = self.o
        fl = o.material == 1
        vs = self._velocity()
        self.xs[fl] = (o.x[fl] + self.dt * vs[fl]).astype(self.r)

    def update_pressure(self):
        """rho*, the pressure update and the sweep's max error (returned)."""
        o, r = self.o, self.r
        fl = o.material == 1
        _, _, q = self._rq()
        den = self._sum((o.m_V[self.j] * self.W(q)).astype(r))
        rho = (self.rho0 * (o.m_V * self.k_w + den)).astype(r)
        self.rho_star = np.where(fl, rho, 0).astype(r)
        e = np.where(fl, np.maximum(rho - self.rho0, r(0)), 0).astype(r)
        o.pressure[fl] = (o.pressure[fl] + self.delta * e[fl]).astype(r)
        return float(e.max()) if fl.any() else 0.0

    def pressure_force(self, react=False):
        """a^p at x* with the current pressures; react: the reactions, added to the dynamic solids' acceleration."""
        o, r = self.o, self.r
        i, j, fj = self.i, self.j, self.fl_j
        d, rn, q = self._rq()
        g = self.gradW(d, rn, q)
        p = o.pressure.astype(r)
        c = (o.m_V[j] * (p[i] + np.where(fj, p[j], p[i]))).astype(r)
        term = (-(c / self.rho0)[:, None] * g).astype(r)
        self.ap = self._sum(term).astype(r)
        self.ap[o.material != 1] = 0
        if react:
            dyn = (~fj) & (o.is_dynamic[j] != 0)
            rb = -(o.density[i][dyn] / o.density[j][dyn])[:, None] * term[dyn]
            np.add.at(o.acceleration, j[dyn], rb.astype(r))
        return self.ap

    def sweep(self):
        self.predict()
        err = self.update_pressure()
        self.pressure_force()
        return err

    def done(self, err, it, eta=MAX_ERROR, min_iterations=MIN_ITERATIONS, max_iterations=MAX_ITERATIONS):
        return (err < eta * float(self.rho0) and it >= min_iterations) or it >= max_iterations

    def pressure_solve(self, **kw):
        it, err = 0, 0.0
        while True:
            err = self.sweep()
            it += 1
            if self.done(err, it, **kw):
                break
        self.last_iterations, self.last_err = it, err
        return it

    def compute_pressure_forces(self):
        self.pressure_force(react=True)

    def update_time_step(self):
        o, r, dt = self.o, self.r, self.dt
        fl = o.material == 1
        vs = self._velocity()
        o.v[fl] = vs[fl]
        sol = (~fl) & (o.is_dynamic != 0)
        o.v[sol] = (o.v[sol] + dt * o.acceleration[sol]).astype(r)
        dyn = o.is_dynamic != 0
        o.x[dyn] = (o.x[dyn] + dt * o.v[dyn]).astype(r)

    def step(self, **kw):
        """sph_base.py:263-271 with the PCISPH substep."""
        o = self.o
        o.initialize_particle_system()
        o.compute_moving_boundary_volume()
        o.compute_densities()
        o.compute_non_pressure_forces()
        self.compute_deltas()
        self.pressure_solve(**kw)
        self.compute_pressure_forces()
        self.update_time_step()
        for oid in o.dyn_ids:
            o.solve_constraints(oid)
            o.enforce_boundary_3D(0)
        o.enforce_boundary_3D(1)
