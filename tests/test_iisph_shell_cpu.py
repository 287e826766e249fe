"""Host logic of IISPHSolver on CPU, with a recording stand-in for the CUDA engine: the solver that
simulationMethod 3 builds, the one-call step, the reference's op sequence of the host-loop structure, and the
refusal of x-slab sharding (Python and the run_simulation.py CLI)."""
import json
import os

import pytest
import torch

from sph_taichi_b200 import SimConfig, scene
from tests.helpers import mixed_scene


class RecordingEngine:
    def __init__(self, params, n_max, n_solid=0, n_bodies=0, device=None):
        self.log = []
        self.err = 1.0
        RecordingEngine.last = self

    def __getattr__(self, name):
        def f(*a, **k):
            self.log.append(name)
            if name in ("check_status", "read_status", "launch_count"):
                return 0
            return None
        return f

    def iisph_op(self, op, arg=0.0, out=None):
        self.log.append(f"iisph:{op}")
        if op == 3:  # pressure_solve_iteration: the sum of the error falls by 10x per sweep
            self.err /= 10.0
            out.fill_(self.err * 64)

    def iisph_solve(self, max_iterations, omega, eta, n_fluid, first_batch):
        self.log.append(f"iisph_solve:{max_iterations}:{omega}:{eta}:{first_batch}")
        return 3, 0.5 * eta

    def iisph_step(self, nsteps, io):
        self.log.append(f"iisph_step:{nsteps}:{io.max_iterations}:{io.omega}:{io.eta}:{io.first_batch}")
        io.iterations, io.avg_err, io.first_batch = 7, 1e-4, 7


@pytest.fixture
def fake_engine(monkeypatch):
    from sph_taichi_b200 import engine
    monkeypatch.setattr(engine, "Engine", RecordingEngine)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    yield


def _iisph_scene():
    sc = mixed_scene(fluid_counts=(4, 4, 4))
    sc["Configuration"]["simulationMethod"] = 3
    sc["Configuration"]["timeStepSize"] = 0.001
    return sc


def _solver():
    from sph_taichi_b200.particle_system import ParticleSystem
    ps = ParticleSystem(SimConfig(_iisph_scene()), device="cpu")
    return ps, ps.build_solver()


def test_method_3_builds_the_iisph_solver(fake_engine):
    from sph_taichi_b200.IISPH import IISPHSolver
    ps, s = _solver()
    assert isinstance(s, IISPHSolver)
    assert "set_iisph" in RecordingEngine.last.log
    assert (s.omega, s.max_iterations, s.max_error, s.surface_tension) == (0.5, 1000, 1e-3, 0.0)
    assert s.dt[None] == pytest.approx(1e-3) and s.device_side_loops
    for name in ("a_ii", "density_deviation", "pressure_accel", "verbose", "last_iterations",
                 "last_avg_density_error"):
        assert hasattr(s, name), name
    for name in ("compute_densities", "compute_non_pressure_forces", "predict_advection", "pressure_solve",
                 "pressure_solve_iteration", "compute_pressure_forces", "advect", "substep"):
        assert callable(getattr(s, name)), name
    assert ps._solver_constants()[-1] == 0.0  # no cohesion in the engine parameters
    sc = _iisph_scene()
    sc["Configuration"]["simulationMethod"] = 2
    from sph_taichi_b200.particle_system import ParticleSystem
    with pytest.raises(NotImplementedError):
        ParticleSystem(SimConfig(sc), device="cpu").build_solver()


def test_step_is_one_library_call(fake_engine):
    ps, s = _solver()
    s.initialize()
    eng = RecordingEngine.last
    eng.log.clear()
    s.step()
    assert eng.log == ["iisph_step:1:1000:0.5:0.001:4"]
    assert (s.last_iterations, s.last_avg_density_error) == (7, 1e-4)
    eng.log.clear()
    s.step(3)  # the next first batch is the last step's sweep count
    assert eng.log == ["iisph_step:3:1000:0.5:0.001:7"]


def test_host_loop_runs_the_reference_op_sequence(fake_engine):
    ps, s = _solver()
    s.device_side_loops = False
    s.initialize()
    eng = RecordingEngine.last
    eng.log.clear()
    n_fluid = ps.fluid_particle_num
    assert n_fluid == 64
    s.step()
    # avg = err * 64 / n_fluid: 0.1, 0.01, 1e-3 (not < 1e-3), 1e-4 -> four sweeps
    assert eng.log == ["neighbor_build", "boundary_volume", "iisph:0", "iisph:1", "iisph:2", "iisph:3", "iisph:3",
                       "iisph:3", "iisph:3", "iisph:4", "iisph:5", "enforce_boundary"], eng.log
    assert s.last_iterations == 4 and s.last_avg_density_error == pytest.approx(1e-4)
    s.device_side_loops = True
    eng.log.clear()
    s.pressure_solve()  # on its own: the device-side loop
    assert eng.log == ["iisph_solve:1000:0.5:0.001:4"] and s.last_iterations == 3


def test_sharding_refuses_iisph_before_any_device_work(monkeypatch):
    from sph_taichi_b200 import engine, slab

    def no_engine(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(engine, "Engine", no_engine)
    with pytest.raises(NotImplementedError, match="IISPH .* is single-GPU"):
        slab.build_sharded(_iisph_scene(), 0, 1, None)
    sc = _iisph_scene()
    sc["Configuration"]["simulationMethod"] = 2
    with pytest.raises(NotImplementedError, match="simulationMethod 2"):
        slab.build_sharded(sc, 0, 1, None)


def test_cli_gpus_refuses_an_iisph_scene(tmp_path):
    """run_simulation.py --gpus 1 on an IISPH scene exits non-zero with the message (host-emulated library)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    from tests.test_slab_gloo_dump import _run
    sc = scene.dam_break_box([6, 6, 6], domain_end=[0.4, 0.4, 0.4], start=[0.1, 0.1, 0.1])
    sc["Configuration"]["simulationMethod"] = 3
    (tmp_path / "iisph.json").write_text(json.dumps(sc))
    res = _run(1, None, ["main", "--", "--scene_file", str(tmp_path / "iisph.json"), "--gpus", "1", "--frames", "1"],
               cwd=str(tmp_path), check=False)
    assert res.returncode != 0 and "single-GPU" in res.stderr, res.stdout[-2000:] + res.stderr[-2000:]
    assert not os.path.exists(tmp_path / "iisph_output")
