"""Numpy restatement of the IISPH formulation of DESIGN.md section 10 (TEST INFRASTRUCTURE ONLY).

Steps 4-7 of an IISPH step (predict_advection, pressure_solve, compute_pressure_forces, advect) on the arrays of an
``oracle.sph_oracle.OracleSim`` (fp32 or fp64), which supplies everything else: the neighbour sort, boundary volumes,
the density pass and the non-pressure forces (with ``surface_tension = 0``), shape matching and the wall clamps.
Neighbour pairs are found with a k-d tree and kept by the reference's exact predicate ``(x_i - x_j).norm() < h``
evaluated in the simulation's precision, so the pair set is the engine's.  The map p -> Ap is available on its own
(``apply_A``) so that tests can assemble A column by column.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

OMEGA, MAX_ITERATIONS, MAX_ERROR = 0.5, 1000, 1e-3


def iisph_oracle(sc, f64=False):
    """An OracleSim of an IISPH scene: the oracle restates methods 0 and 4, and IISPH's density pass and non-pressure
    forces are DFSPH's without cohesion, so it is built as a DFSPH scene with surface_tension = 0."""
    import copy

    from oracle.sph_oracle import OracleSim
    sc = copy.deepcopy(sc)
    sc["Configuration"]["simulationMethod"] = 4
    o = OracleSim(sc, f64=f64)
    o.P.surface_tension = 0.0
    return o


class IisphRef:
    def __init__(self, o):
        self.o = o
        self.r = o.real
        self.dt = self.r(o.P.dt)
        self.rho0 = self.r(o.P.density0)
        self.h = self.r(o.support_radius)
        self.k_dw = self.r(6.0 * 8 / np.pi / float(o.support_radius) ** 3)
        self.last_iterations, self.last_avg = 0, 0.0

    # ---- geometry ------------------------------------------------------------------------------------------------
    def pairs(self):
        """(i, j, gradW(x_i - x_j)) for every fluid i and neighbour j != i."""
        o, r = self.o, self.r
        x = o.x.astype(r)
        tree = cKDTree(x.astype(np.float64))
        pr = tree.query_pairs(float(self.h) * (1 + 1e-5), output_type="ndarray")
        i = np.concatenate([pr[:, 0], pr[:, 1]])
        j = np.concatenate([pr[:, 1], pr[:, 0]])
        d = x[i] - x[j]
        rn = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        keep = (rn < self.h) & (o.material[i] == 1)
        i, j, d, rn = i[keep], j[keep], d[keep], rn[keep]
        q = rn / self.h
        ok = (rn > r(1e-5)) & (q <= 1)
        safe = np.where(ok, rn, r(1))
        gq = d / (safe * self.h)[:, None]
        f = r(1) - q
        res = np.where(q <= r(0.5), self.k_dw * q * (r(3) * q - r(2)), self.k_dw * (-f * f))
        g = np.where(ok[:, None], res[:, None] * gq, r(0)).astype(r)
        fl_j = o.material[j] == 1
        self.i, self.j, self.g, self.fl_j = i, j, g, fl_j
        return i, j, g

    def _sum(self, vals):
        out = np.zeros((self.o.n,) + vals.shape[1:], dtype=vals.dtype)
        np.add.at(out, self.i, vals)
        return out

    # ---- steps 4-7 -----------------------------------------------------------------------------------------------
    def predict_advection(self):
        o, r, dt, rho0 = self.o, self.r, self.dt, self.rho0
        self.pairs()
        fl = o.material == 1
        o.v[fl] = (o.v[fl] + dt * o.acceleration[fl]).astype(r)  # v*
        i, j, g, fj = self.i, self.j, self.g, self.fl_j
        psi = (rho0 * o.m_V).astype(r)
        rho = o.density
        div = self._sum(psi[j] * np.einsum("ij,ij->i", o.v[i] - o.v[j], g))
        self.s = np.where(fl, rho0 - rho - dt * div, 0).astype(r)
        pg = psi[j][:, None] * g
        cf = self._sum(np.where(fj[:, None], pg, 0))
        cb = self._sum(np.where(fj[:, None], 0, pg))
        sq = self._sum(np.where(fj, psi[j] * np.einsum("ij,ij->i", g, g), 0))
        inv_r2 = np.where(fl, r(1) / (rho * rho), 0).astype(r)
        c = -inv_r2[:, None] * cf - (inv_r2 + r(1) / (rho0 * rho0))[:, None] * cb
        self.a_ii = np.where(fl, dt * dt * (np.einsum("ij,ij->i", cf + cb, c) - psi * inv_r2 * sq), 0).astype(r)
        o.pressure[fl] = (r(0.5) * o.pressure[fl]).astype(r)

    def accel(self, p, react=False):
        """a^p for pressures p (solids: 0); react: also the reactions, added to the dynamic solids' acceleration."""
        o, r, rho0 = self.o, self.r, self.rho0
        i, j, g, fj = self.i, self.j, self.g, self.fl_j
        psi = (rho0 * o.m_V).astype(r)
        fl = o.material == 1
        dp = np.where(fl, p / (o.density * o.density), 0).astype(r)
        coef = np.where(fj, dp[i] + dp[j], dp[i] + p[i] / (rho0 * rho0))
        term = -(psi[j] * coef)[:, None] * g
        ap = self._sum(term)
        if react:
            dyn = (~fj) & (o.is_dynamic[j] != 0)
            rb = -(o.density[i][dyn] / o.density[j][dyn])[:, None] * term[dyn]
            np.add.at(o.acceleration, j[dyn], rb.astype(r))
        return ap.astype(r)

    def apply_A(self, ap):
        o, r, rho0, dt = self.o, self.r, self.rho0, self.dt
        i, j, g, fj = self.i, self.j, self.g, self.fl_j
        psi = (rho0 * o.m_V).astype(r)
        apj = np.where(fj[:, None], ap[j], 0)
        return (dt * dt * self._sum(psi[j] * np.einsum("ij,ij->i", ap[i] - apj, g))).astype(r)

    def sweep(self, omega=OMEGA):
        o, r = self.o, self.r
        fl = o.material == 1
        p = o.pressure.astype(r)
        self.ap = self.accel(p)
        Ap = self.apply_A(self.ap)
        big = np.abs(self.a_ii) > r(1e-6)
        a_safe = np.where(big, self.a_ii, r(1))
        pn = np.where(big, np.maximum(p + r(omega) * (self.s - Ap) / a_safe, r(0)), r(0)).astype(r)
        o.pressure[fl] = pn[fl]
        act = fl & (pn > 0)
        self.Ap = Ap
        err = float(np.sum(np.abs(Ap[act].astype(np.float64) - self.s[act]) / float(self.rho0)))
        return err / int(fl.sum())

    def pressure_solve(self, max_iterations=MAX_ITERATIONS, eta=MAX_ERROR):
        it, avg = 0, 0.0
        while it < max_iterations:
            avg = self.sweep()
            it += 1
            if avg < eta:
                break
        self.last_iterations, self.last_avg = it, avg
        return it

    def compute_pressure_forces(self):
        o = self.o
        fl = o.material == 1
        self.ap = self.accel(o.pressure.astype(self.r), react=True)
        o.acceleration[fl] = self.ap[fl]

    def advect(self):
        o, dt = self.o, self.dt
        dyn = o.is_dynamic != 0
        o.v[dyn] = (o.v[dyn] + dt * o.acceleration[dyn]).astype(self.r)
        o.x[dyn] = (o.x[dyn] + dt * o.v[dyn]).astype(self.r)

    def step(self):
        """sph_base.py:263-271 with the IISPH substep."""
        o = self.o
        o.initialize_particle_system()
        o.compute_moving_boundary_volume()
        o.compute_densities()
        o.compute_non_pressure_forces()
        self.predict_advection()
        self.pressure_solve()
        self.compute_pressure_forces()
        self.advect()
        for oid in o.dyn_ids:
            o.solve_constraints(oid)
            o.enforce_boundary_3D(0)
        o.enforce_boundary_3D(1)
