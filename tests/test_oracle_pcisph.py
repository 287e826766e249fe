"""The PCISPH restatement of tests/pcisph_ref.py on CPU: one sweep against a dense all-pairs evaluation, delta against
an independent fp64 evaluation, fp32 against fp64, the loop rule, and the converged state of the loop."""
import numpy as np
import pytest

from sph_taichi_b200.PCISPH import scaling_factor
from tests.helpers import jitter, mixed_scene, order_by_x0
from tests.pcisph_ref import PcisphRef, pcisph_oracle


def _state(f64, squeeze=0.93, seed=4, dt=0.001):
    sc = mixed_scene(fluid_counts=(7, 7, 7))
    sc["Configuration"]["simulationMethod"] = 1
    sc["Configuration"]["timeStepSize"] = dt
    o = pcisph_oracle(sc, f64=f64)
    jitter(o, 0.002, seed=seed)
    fl = o.material == 1
    c = o.x[fl].mean(axis=0)
    o.x[fl] = ((o.x[fl] - c) * o.real(squeeze) + c).astype(o.real)
    o.initialize()
    o.compute_densities()
    o.compute_non_pressure_forces()
    ref = PcisphRef(o, scaling_factor(dt, o.particle_radius))
    ref.compute_deltas()
    return o, ref


def test_one_sweep_against_a_dense_restatement():
    o, ref = _state(f64=True)
    ref.sweep()
    fl = o.material == 1
    rho0, dt, h = 1000.0, 0.001, float(o.support_radius)
    # x* of the dense evaluation from scratch: v* = v + dt a^np (a^p = 0 in the first sweep)
    xs = np.where(fl[:, None], o.x + dt * (o.v + dt * ref.anp), o.x)
    assert np.allclose(ref.xs, xs, rtol=0, atol=1e-12)
    d = xs[:, None, :] - xs[None, :, :]
    r = np.sqrt((d * d).sum(-1))
    x0 = o.x.astype(np.float64)
    d0 = x0[:, None, :] - x0[None, :, :]
    nb = (np.sqrt((d0 * d0).sum(-1)) < h) & ~np.eye(o.n, dtype=bool) & fl[:, None]  # the lists, at x^t
    k = 8 / np.pi / h ** 3
    q = r / h
    W = np.where(q <= 0.5, k * (6 * q ** 3 - 6 * q ** 2 + 1), 2 * k * np.clip(1 - q, 0, None) ** 3)
    rho = rho0 * (o.m_V * k + (np.where(nb, W, 0) * o.m_V[None, :]).sum(1))
    assert np.allclose(ref.rho_star[fl], rho[fl], rtol=1e-12)
    e = np.maximum(rho - rho0, 0)
    assert float(e[fl].max()) > 10.0  # compressed: the first sweep does not meet eta
    p = np.where(fl, ref.delta * e, 0)
    assert np.allclose(o.pressure[fl], p[fl], rtol=1e-12)
    gs = np.where(q <= 0.5, 6 * k * q * (3 * q - 2), -6 * k * (1 - q) ** 2) / np.where(r > 1e-5, r * h, 1.0)
    g = np.where((nb & (r > 1e-5) & (q <= 1))[..., None], gs[..., None] * d, 0.0)
    pj = np.where(fl[None, :], p[None, :], p[:, None])  # the mirrored pressure of a solid neighbour
    ap = -np.einsum("j,ij,ijk->ik", o.m_V, p[:, None] + pj, g) / rho0
    scale = np.abs(ap[fl]).max()
    assert scale > 1.0
    assert np.allclose(ref.ap[fl], ap[fl], rtol=0, atol=1e-10 * scale)


def test_delta_against_a_larger_lattice_cube():
    """delta sums the lattice nodes inside the support; a cube of 7^3 nodes around them adds only zero terms."""
    for radius, dt in ((0.01, 0.001), (0.02, 4e-4)):
        d, h = 2 * radius, 4 * radius
        a = np.arange(-3, 4) * d
        x = np.array(np.meshgrid(a, a, a, indexing="ij")).reshape(3, -1).T
        r = np.linalg.norm(x, axis=1)
        keep = r > 0
        x, r = x[keep], r[keep]
        q = r / h
        k_dw = 48 / np.pi / h ** 3
        f = np.where(q <= 0.5, k_dw * q * (3 * q - 2), np.where(q < 1, -k_dw * (1 - q) ** 2, 0.0))
        g = f[:, None] * x / (r * h)[:, None]
        beta = 2 * (dt * 0.8 * d ** 3) ** 2
        expect = 1 / (beta * (np.dot(g.sum(0), g.sum(0)) + (g * g).sum()))
        assert scaling_factor(dt, radius) == pytest.approx(expect, rel=1e-12)
    # delta scales as 1 / dt^2
    assert scaling_factor(5e-4, 0.01) == pytest.approx(4 * scaling_factor(1e-3, 0.01), rel=1e-12)


def test_fp32_against_fp64():
    (o32, r32), (o64, r64) = _state(False), _state(True)
    k32, k64 = order_by_x0(o32.x_0), order_by_x0(o64.x_0)  # the two precisions may sort a cell differently
    assert np.array_equal(o32.material[k32], o64.material[k64])
    fl = o64.material[k64] == 1

    def rel(a, b):
        a, b = a[k32][fl].astype(np.float64), b[k64][fl]
        return float(np.abs(a - b).max() / np.abs(b).max())

    for _ in range(2):  # the second sweep starts from non-zero pressures and a^p
        e32, e64 = r32.sweep(), r64.sweep()
        assert rel(r32.rho_star, r64.rho_star) < 2e-6
        assert abs(e32 - e64) <= 2e-6 * 1000.0
        assert rel(o32.pressure, o64.pressure) < 5e-4
        assert rel(r32.ap, r64.ap) < 5e-4


class _Scripted(PcisphRef):
    """The loop rule alone: each sweep returns the next scripted max error."""

    def __init__(self, errs):
        self.errs = list(errs)
        self.n = 0

    def sweep(self):
        self.n += 1
        return self.errs.pop(0)

    rho0 = np.float32(1000.0)


def test_loop_rule():
    # at least 3 sweeps even when the first already meets eta (1 % rho0 = 10)
    s = _Scripted([1.0, 1.0, 1.0, 1.0])
    assert s.pressure_solve() == 3 and s.n == 3
    # after the third, the first sweep under eta stops the loop (10.0 itself does not)
    s = _Scripted([50.0, 30.0, 20.0, 10.0, 9.99, 1.0])
    assert s.pressure_solve() == 5 and s.last_err == 9.99
    # the cap
    s = _Scripted([50.0] * 20)
    assert s.pressure_solve(max_iterations=7) == 7 and s.n == 7


def test_converged_state_meets_eta():
    """A free fluid block squeezed by 9 % (rho up to 1.11 rho0): the loop converges well past its minimum, and in the
    converged fp64 state the max predicted density error is below eta rho0.  (Larger squeezes, and fluid started inside
    a solid's support, are outside the loop's reach: the error clamp lets the pressure only grow, and it oscillates to
    the cap -- DESIGN.md section 11.)"""
    sc = mixed_scene(fluid_counts=(7, 7, 7), with_static=False, with_dynamic=False)
    sc["Configuration"]["simulationMethod"] = 1
    sc["Configuration"]["timeStepSize"] = 0.001
    o = pcisph_oracle(sc, f64=True)
    jitter(o, 0.001, seed=4)
    fl = o.material == 1
    c = o.x[fl].mean(axis=0)
    o.x[fl] = (o.x[fl] - c) * 0.91 + c
    o.initialize()
    o.compute_densities()
    o.compute_non_pressure_forces()
    assert float(o.density[fl].max()) > 1100.0
    ref = PcisphRef(o, scaling_factor(0.001, o.particle_radius))
    ref.compute_deltas()
    it = ref.pressure_solve()
    assert 10 < it < 1000 and ref.last_err < 10.0, (it, ref.last_err)
    e = np.maximum(ref.rho_star[fl] - 1000.0, 0)
    assert float(e.max()) < 10.0 and float(e.max()) == ref.last_err
    assert float(o.pressure[fl].max()) > 0.0
