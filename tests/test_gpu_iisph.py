"""IISPH (simulationMethod 3, DESIGN.md section 10): CUDA engine against the numpy restatement of tests/iisph_ref.py
on top of the CPU oracle.

Per-kernel parity starts every kernel from the engine's own inputs (the restatement is given the engine's state
before the kernel), so each comparison measures one kernel; tolerances are those of tests/test_gpu_dfsph.py.  The
Jacobi loop stops on an averaged error, so an fp32 difference in the last digit can change a sweep count by one; the
whole-step test then accepts a trajectory within the solver's own tolerance, as the DFSPH test does."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.helpers import jitter, mixed_scene, order_by_x0
from tests.iisph_ref import IisphRef, iisph_oracle

pytestmark = pytest.mark.gpu
REL = 5e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _maxrel(a, b):
    scale = max(float(np.abs(b).max()), 1e-30)
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max()) / scale


def _iisph(sc, dt=0.001):
    sc["Configuration"]["simulationMethod"] = 3
    sc["Configuration"]["timeStepSize"] = dt
    return sc


def _pair(sc, seed=None, amp=0.002, squeeze=1.0):
    from sph_taichi_b200 import ParticleSystem, SimConfig
    o = iisph_oracle(sc)
    ps = ParticleSystem(SimConfig(sc))
    if seed is not None:
        jitter(o, amp, seed=seed)
        fl = o.material == 1
        c = o.x[fl].mean(axis=0)
        o.x[fl] = ((o.x[fl] - c) * np.float32(squeeze) + c).astype(np.float32)
        ps.x.from_numpy(o.x)
        ps.v.from_numpy(o.v)
    return o, ps, ps.build_solver()


def _kernel_chain(o, ps, s, expect_reactions, overflow=False):
    """Every IISPH kernel once, each compared from identical inputs."""
    ref = IisphRef(o)
    fl = o.material == 1
    rho0 = 1000.0
    o.pressure[fl] = np.linspace(0, 2000, int(fl.sum()), dtype=np.float32)  # a previous step's pressure
    ps.pressure.from_numpy(o.pressure)
    o.initialize(); s.initialize()
    fl = o.material == 1  # the sort permuted the arrays
    o.compute_densities(); s.compute_densities()
    if overflow:
        assert ps._engine.neighbor_stats()["overflow"] > 100
    assert np.array_equal(ps.x.to_numpy(), o.x)
    assert _maxrel(ps.density.to_numpy(), o.density) < REL
    assert float(o.density[fl].max()) > 1050.0  # genuinely compressed: the solver has work to do
    o.density[:] = ps.density.to_numpy()
    o.compute_non_pressure_forces(); s.compute_non_pressure_forces()
    assert _maxrel(ps.acceleration.to_numpy(), o.acceleration) < REL
    o.acceleration[:] = ps.acceleration.to_numpy()
    assert np.array_equal(ps.pressure.to_numpy(), o.pressure)
    # predict_advection
    ref.predict_advection(); s.predict_advection()
    assert _maxrel(ps.v.to_numpy(), o.v) < REL
    a_g, s_g = s.a_ii.to_numpy(), s.density_deviation.to_numpy()
    assert float((np.abs(ref.a_ii[fl]) > 1e-6).mean()) > 0.9
    assert _maxrel(a_g[fl], ref.a_ii[fl]) < 5 * REL
    assert np.abs(s_g[fl] - ref.s[fl]).max() / rho0 < 5 * REL  # s_i is a density: its error is the density error
    assert np.array_equal(ps.pressure.to_numpy()[fl], o.pressure[fl])  # warm start: exactly 0.5 p
    ref.a_ii[:], ref.s[:] = a_g, s_g
    # one sweep
    err = s.pressure_solve_iteration()
    e_ref = ref.sweep()
    assert _maxrel(s.pressure_accel.to_numpy()[fl], ref.ap[fl]) < 5 * REL
    p_g = ps.pressure.to_numpy()
    assert int((p_g[fl] > 0).sum()) > 0
    assert _maxrel(p_g[fl], o.pressure[fl]) < 10 * REL
    assert abs(err - e_ref) <= 1e-3 * abs(e_ref) + 1e-7, (err, e_ref)
    o.pressure[:] = p_g
    # pressure forces + reactions
    acc0 = o.acceleration.copy()
    ref.compute_pressure_forces(); s.compute_pressure_forces()
    a_g = ps.acceleration.to_numpy()
    assert _maxrel(a_g[fl], o.acceleration[fl]) < 5 * REL
    dyn = (o.material == 0) & (o.is_dynamic == 1)
    if expect_reactions:
        assert np.abs(o.acceleration[dyn] - acc0[dyn]).max() > 0.1  # reactions present
        assert _maxrel(a_g[dyn] - acc0[dyn], o.acceleration[dyn] - acc0[dyn]) < 10 * REL
    o.acceleration[:] = a_g
    o.v[:] = ps.v.to_numpy()
    ref.advect(); s.advect()
    assert _maxrel(ps.x.to_numpy(), o.x) < 1e-6
    with pytest.raises(RuntimeError, match="stale"):
        s.predict_advection()


def test_iisph_per_kernel_parity():
    from sph_taichi_b200.IISPH import IISPHSolver
    o, ps, s = _pair(_iisph(mixed_scene()), seed=2, squeeze=0.93)
    assert isinstance(s, IISPHSolver)
    _kernel_chain(o, ps, s, expect_reactions=True)


def test_iisph_kernels_on_overfull_neighbour_lists():
    """The same kernels on a state with > 96 neighbours per particle: the 27-cell fallback of the list walk."""
    o, ps, s = _pair(_iisph(mixed_scene(with_dynamic=False)), seed=3, squeeze=0.6)
    _kernel_chain(o, ps, s, expect_reactions=False, overflow=True)


def _dam(counts=(14, 18, 12)):
    from sph_taichi_b200 import scene
    return _iisph(scene.dam_break_box(list(counts), domain_end=[0.8, 0.8, 0.6], start=[0.06, 0.06, 0.06]))


def test_iisph_steps_vs_oracle():
    """Whole steps of a dam break against the restatement: the loop iterates (more than one sweep per step)."""
    o, ps, s = _pair(_dam(), seed=11, amp=0.002, squeeze=0.93)
    ref = IisphRef(o)
    o.initialize(); s.initialize()
    counts_o, counts_g = [], []
    for _ in range(25):
        ref.step(); s.step()
        counts_o.append(ref.last_iterations)
        counts_g.append(s.last_iterations)
    assert ps._engine.check_status() == 0
    assert max(counts_o) >= 2, counts_o
    ko, kg = order_by_x0(o.x_0), order_by_x0(ps.x_0.to_numpy())
    err = np.abs(ps.x.to_numpy()[kg] - o.x[ko]).max() / 0.02
    same = counts_o == counts_g
    assert err < (2e-3 if same else 5e-2), (err, same, counts_o, counts_g)


def test_device_side_loop_runs_the_same_sweeps_as_the_host_loop():
    """sph_iisph_step only moves the loop condition: same sweeps, same counts, bit-identical state."""
    runs = []
    for dev_loops in (True, False):
        _, ps, s = _pair(_dam(), seed=11, amp=0.002, squeeze=0.93)
        s.device_side_loops = dev_loops
        s.initialize()
        counts = []
        for _ in range(6):
            s.step()
            counts.append(s.last_iterations)
        assert ps._engine.check_status() == 0
        runs.append((counts, ps.x.to_numpy().copy(), ps.v.to_numpy().copy(), ps.pressure.to_numpy().copy()))
    assert runs[0][0] == runs[1][0]
    assert max(runs[0][0]) >= 2, runs[0][0]
    for a, b in zip(runs[0][1:], runs[1][1:]):
        assert np.array_equal(a, b)


def _tank(nx=10, ny=16, dt=0.001):
    """A fluid column of nx x ny x nx particles (d = 0.02 m) in a tank of static blocks two layers thick: a floor
    under it and four walls one spacing away from it, higher than the column."""
    from sph_taichi_b200 import scene
    d = 0.02
    hi = 0.1 + nx * d  # first wall layer on the far sides
    top = 0.1 + (ny + 1.5) * d

    def blk(oid, s, e):
        return {"objectId": oid, "start": s, "end": e, "translation": [0.0] * 3, "scale": [1, 1, 1],
                "velocity": [0.0] * 3, "density": 1000.0, "color": [255] * 3, "isDynamic": False}

    sc = scene.dam_break_box([nx, ny, nx], domain_end=[hi + 0.2, 0.1 + (ny + 4) * d, hi + 0.2], start=[0.1] * 3)
    sc["RigidBlocks"] = [blk(1, [0.06, 0.06, 0.06], [hi + 1.5 * d, 0.06 + 1.5 * d, hi + 1.5 * d]),
                         blk(2, [0.06, 0.10, 0.06], [0.06 + 1.5 * d, top, hi + 1.5 * d]),
                         blk(3, [hi, 0.10, 0.06], [hi + 1.5 * d, top, hi + 1.5 * d]),
                         blk(4, [0.10, 0.10, 0.06], [hi - 0.5 * d, top, 0.06 + 1.5 * d]),
                         blk(5, [0.10, 0.10, hi], [hi - 0.5 * d, top, hi + 1.5 * d])]
    return _iisph(sc, dt)


def _bottom_ratio(ps, nx=10, ny=16, d=0.02):
    """Median pressure of the bottom layer's inner particles over rho0 g H (H = ny d), and the kinetic energy per
    unit mass."""
    x, v, p = ps.x.to_numpy(), ps.v.to_numpy(), ps.pressure.to_numpy()
    fl = ps.material.to_numpy() == 1
    y, c = x[fl, 1], 0.1 + (nx - 1) * d / 2
    inner = (np.abs(x[fl, 0] - c) < (nx / 2 - 2) * d) & (np.abs(x[fl, 2] - c) < (nx / 2 - 2) * d)
    bottom = inner & (y < y.min() + 0.5 * d)
    return float(np.median(p[fl][bottom])) / (1000.0 * 9.81 * ny * d), float((v[fl] ** 2).sum(1).mean() / 2)


def test_hydrostatic_column_at_rest():
    """A 10 x 16 x 10 column in a tank, settled, against the hydrostatic pressure rho0 g H, H = 16 d = 0.32 m.

    Expected ratio p_bottom / (rho0 g H).  By momentum balance a column at rest carries rho0 g times the depth of the
    bottom layer's centres below the free surface.  Two SPH effects make that depth smaller than H:
    * the rest spacing is not d.  A particle's volume is m_V = 0.8 d^3, so the fluid reaches rho0 at the spacing
      s = 0.8^(1/3) d = 0.928 d: the column settles 7 % shorter than its initial lattice.  The measured layers agree:
      bottom centres at y = 0.1069, top centres at y = 0.3817, 15 spacings of 0.0183 m;
    * the depth of the bottom centres is 15.5 spacings (the surface sits half a spacing above the top centres), so
      the expected ratio is 15.5 s / (16 d) = 0.90.  The surface layer is particle deficient (rho < rho0, p clamped
      to 0), which lowers the effective surface a little further.
    Measured on one H100 80GB HBM3: with a converged loop (eta = 1e-5, ~70 sweeps per step) the ratio is 0.875 +-
    0.010 over the last 1000 of 2000 steps (dt = 1e-3) (16 x 24 x 16: 0.838 +- 0.029), i.e. 0.97 x the estimate above.
    With the reference's criterion (avg < 1e-3: one or two sweeps per step, warm start 0.5 p) the column comes to the
    same rest (kinetic energy < 1e-4 J/kg) and the same mean (0.856 over the last 1000 steps) but a single snapshot
    scatters by +-0.17: the loop stops with a residual s - Ap of the order of a_ii p, which moves the pressure of
    single particles from step to step.  So the offset below 1 is the discretisation, not the solver (it does not
    shrink with eta), and the bounds are: converged, one snapshot in [0.82, 0.95]; default criterion, the mean of 40
    snapshots in [0.75, 1.0] (the standard error of that mean is about 0.03)."""
    from sph_taichi_b200 import ParticleSystem, SimConfig
    for eta in (1e-5, 1e-3):
        ps = ParticleSystem(SimConfig(_tank()))
        s = ps.build_solver()
        s.max_error = eta
        s.initialize()
        s.step(1000)  # 1 s: settled
        ratios, kes = [], []
        for _ in range(40):  # the next second, a snapshot every 25 steps
            s.step(25)
            r, ke = _bottom_ratio(ps)
            ratios.append(r)
            kes.append(ke)
        assert ps._engine.check_status() == 0
        assert max(kes) < 1e-3 and np.median(kes) < 2e-4, (eta, kes)  # at rest: |v| ~ 1 cm/s
        if eta < 1e-4:
            assert s.last_iterations > 10  # the loop really converges further than the default one
            assert all(0.82 < r < 0.95 for r in ratios), ratios
        else:
            assert s.last_iterations <= 5
            assert 0.75 < float(np.mean(ratios)) < 1.0, ratios


def test_iisph_dragon_bath_full_size():
    """The dragon_bath_iisph scene at full size: a few steps with a finite state inside the domain."""
    from sph_taichi_b200 import ParticleSystem, SimConfig, scene
    ps = ParticleSystem(SimConfig(scene.dragon_bath_iisph()))
    s = ps.build_solver()
    s.initialize()
    its = []
    for _ in range(8):
        s.step()
        its.append(s.last_iterations)
    assert ps._engine.check_status() == 0
    d = ps.dump(0)
    assert d["position"].shape == (423500, 3) and np.isfinite(d["velocity"]).all()
    pad = np.float32(0.04)
    hi = (np.array([5.0, 3.0, 2.0]) - 0.04).astype(np.float32)
    assert (d["position"] >= pad).all() and (d["position"] <= hi).all()
    assert max(its) <= 1000, its


def test_cli_writes_the_ply_series(tmp_path):
    """run_simulation.py on a small IISPH scene writes the PLY series through build_solver."""
    import json

    from sph_taichi_b200 import scene
    sc = _iisph(scene.dam_break_box([8, 8, 8], domain_end=[0.5, 0.5, 0.5], start=[0.1, 0.1, 0.1]), dt=0.004)
    sc["Configuration"]["exportPly"] = True
    (tmp_path / "iisph_cli.json").write_text(json.dumps(sc))
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "run_simulation.py"), "--scene_file", "iisph_cli.json",
                          "--frames", "9", "--quiet"], cwd=str(tmp_path), env=env, capture_output=True, text=True,
                         timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    names = sorted(os.listdir(tmp_path / "iisph_cli_output"))
    assert names == [f"particle_object_0_{k:06}.ply" for k in range(3)], names
