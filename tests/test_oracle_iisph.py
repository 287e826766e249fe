"""The IISPH restatement of tests/iisph_ref.py on CPU: a dense all-pairs restatement of the source term and of the
operator p -> Ap, the matrix A assembled column by column with unit pressures, fp32 against fp64, and the Jacobi
loop on a compressed block."""
import numpy as np

from tests.helpers import jitter, mixed_scene, order_by_x0
from tests.iisph_ref import IisphRef, iisph_oracle


def _state(f64, squeeze=0.9, seed=4):
    sc = mixed_scene(fluid_counts=(7, 7, 7))
    sc["Configuration"]["simulationMethod"] = 3
    sc["Configuration"]["timeStepSize"] = 0.001
    o = iisph_oracle(sc, f64=f64)
    jitter(o, 0.002, seed=seed)
    fl = o.material == 1
    c = o.x[fl].mean(axis=0)
    o.x[fl] = ((o.x[fl] - c) * o.real(squeeze) + c).astype(o.real)
    o.initialize()
    o.compute_densities()
    o.compute_non_pressure_forces()
    ref = IisphRef(o)
    ref.predict_advection()
    return o, ref


def _dense(o):
    """All pairs in fp64: gradW(x_i - x_j) [n, n, 3] and the neighbour mask of fluid rows."""
    x = o.x.astype(np.float64)
    h = float(o.support_radius)
    k_dw = 6.0 * 8 / np.pi / h ** 3
    d = x[:, None, :] - x[None, :, :]
    r = np.sqrt((d * d).sum(-1))
    q = r / h
    nb = (r < h) & ~np.eye(len(x), dtype=bool) & (o.material == 1)[:, None]
    s = np.where(q <= 0.5, k_dw * q * (3 * q - 2), -k_dw * (1 - q) ** 2) / np.where(r > 1e-5, r * h, 1.0)
    g = np.where((nb & (r > 1e-5))[..., None], s[..., None] * d, 0.0)
    return g, nb


def test_source_term_and_A_against_a_dense_restatement():
    o, ref = _state(f64=True)
    fl = o.material == 1
    g, nb = _dense(o)
    rho0, dt = 1000.0, 0.001
    psi = rho0 * o.m_V
    fj = fl[None, :] & nb
    bj = (~fl)[None, :] & nb
    div = np.einsum("j,ijk,ijk->i", psi, o.v[:, None, :] - o.v[None, :, :], g)
    s = np.where(fl, rho0 - o.density - dt * div, 0.0)
    assert float(np.abs(s).max()) > 1.0
    assert np.allclose(ref.s, s, rtol=0, atol=1e-9 * np.abs(s).max())

    def A(p):
        dp = np.where(fl, p / o.density ** 2, 0.0)
        cf = np.where(fj, dp[:, None] + dp[None, :], 0) + np.where(bj, (dp + p / rho0 ** 2)[:, None], 0)
        ap = -np.einsum("ij,j,ijk->ik", cf, psi, g)
        ap[~fl] = 0
        return dt * dt * (np.einsum("j,ij,ijk,ijk->i", psi, fj, ap[:, None, :] - ap[None, :, :], g)
                          + np.einsum("j,ij,ik,ijk->i", psi, bj, ap, g))

    idx = np.nonzero(fl)[0]
    cols = []
    for k in idx:  # column by column with unit pressures
        e = np.zeros(o.n)
        e[k] = 1.0
        cols.append(ref.apply_A(ref.accel(e))[idx])
    M = np.array(cols).T
    assert np.allclose(np.diag(M), ref.a_ii[idx], rtol=1e-9, atol=1e-9 * np.abs(ref.a_ii).max())
    assert float(np.abs(np.diag(M)).min()) > 0 and float(np.abs(M - np.diag(np.diag(M))).max()) > 0
    rng = np.random.default_rng(0)
    p = np.zeros(o.n)
    p[idx] = rng.uniform(0, 3000, len(idx))
    Ap = ref.apply_A(ref.accel(p))
    scale = np.abs(Ap).max()
    assert np.allclose(Ap[idx], M @ p[idx], rtol=0, atol=1e-9 * scale)
    assert np.allclose(Ap, np.where(fl, A(p), 0.0), rtol=0, atol=1e-9 * scale)


def test_fp32_against_fp64():
    (o32, r32), (o64, r64) = _state(False), _state(True)
    k32, k64 = order_by_x0(o32.x_0), order_by_x0(o64.x_0)  # the two precisions may sort a cell differently
    assert np.array_equal(o32.material[k32], o64.material[k64])
    fl = o64.material[k64] == 1

    def rel(a, b):
        a, b = a[k32][fl].astype(np.float64), b[k64][fl]
        return float(np.abs(a - b).max() / np.abs(b).max())

    assert rel(r32.a_ii, r64.a_ii) < 5e-5
    assert float(np.abs(r32.s[k32][fl] - r64.s[k64][fl]).max()) / 1000.0 < 5e-5
    r32.sweep(), r64.sweep()
    e32, e64 = r32.sweep(), r64.sweep()  # the second sweep starts from non-zero pressures
    assert rel(r32.ap, r64.ap) < 5e-4
    assert rel(o32.pressure, o64.pressure) < 5e-4
    assert abs(e32 - e64) <= 1e-3 * e64


def test_jacobi_converges_on_a_compressed_block():
    o, ref = _state(True, squeeze=0.9)
    fl = o.material == 1
    assert float(o.density[fl].max()) > 1050.0
    it = ref.pressure_solve()
    assert 2 <= it < 1000 and ref.last_avg < 1e-3, (it, ref.last_avg)
    # The converged pressures satisfy A p = s on the active set to the loop's tolerance eta = 1e-3.  The loop's own
    # error is taken from Ap of a sweep's INPUT pressures; this re-evaluates A p on the final pressures and the final
    # active set, which the last relaxation step moved closer to s (8.8e-4 here against the loop's last 9.9e-4).
    act = fl & (o.pressure > 0)
    Ap = ref.apply_A(ref.accel(o.pressure.copy()))
    assert int(act.sum()) > 50
    assert float(np.abs(Ap[act] - ref.s[act]).sum()) / 1000.0 / int(fl.sum()) < 1e-3
