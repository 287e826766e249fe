"""Host logic of PCISPHSolver on CPU, with a recording stand-in for the CUDA engine: the solver that simulationMethod 1
builds, the one-call step, the op sequence of the legacy host-loop structure with its loop rule, and the refusal of
x-slab sharding (Python and the run_simulation.py CLI)."""
import json
import os

import numpy as np
import pytest
import torch

from sph_taichi_b200 import SimConfig, scene
from tests.helpers import mixed_scene


class RecordingEngine:
    errs = []

    def __init__(self, params, n_max, n_solid=0, n_bodies=0, device=None):
        self.log = []
        RecordingEngine.last = self

    def __getattr__(self, name):
        def f(*a, **k):
            self.log.append(name)
            if name in ("check_status", "read_status", "launch_count"):
                return 0
            return None
        return f

    def pcisph_op(self, op, arg=0.0, out=None):
        self.log.append(f"pcisph:{op}")
        if op == 3:  # pci_update_pressure: the next scripted max error, as float bits
            out.view(torch.float32).fill_(RecordingEngine.errs.pop(0))

    def pcisph_solve(self, delta, eta, min_iterations, max_iterations, first_batch):
        self.log.append(f"pcisph_solve:{eta}:{min_iterations}:{max_iterations}:{first_batch}")
        return 5, 0.5

    def pcisph_step(self, nsteps, io):
        self.log.append(f"pcisph_step:{nsteps}:{io.eta}:{io.min_iterations}:{io.max_iterations}:{io.first_batch}")
        self.delta = io.delta
        io.iterations, io.max_err, io.first_batch = 7, 4.5, 7


@pytest.fixture
def fake_engine(monkeypatch):
    from sph_taichi_b200 import engine
    monkeypatch.setattr(engine, "Engine", RecordingEngine)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    yield


def _pcisph_scene():
    sc = mixed_scene(fluid_counts=(4, 4, 4))
    sc["Configuration"]["simulationMethod"] = 1
    sc["Configuration"]["timeStepSize"] = 0.001
    return sc


def _solver():
    from sph_taichi_b200.particle_system import ParticleSystem
    ps = ParticleSystem(SimConfig(_pcisph_scene()), device="cpu")
    return ps, ps.build_solver()


def test_method_1_builds_the_pcisph_solver(fake_engine):
    from sph_taichi_b200.PCISPH import PCISPHSolver, scaling_factor
    ps, s = _solver()
    assert isinstance(s, PCISPHSolver)
    assert "set_pcisph" in RecordingEngine.last.log
    assert (s.max_error, s.sub_max_iteration, s.max_iterations, s.surface_tension) == (0.01, 3, 1000, 0.0)
    assert s.dt[None] == pytest.approx(1e-3) and s.device_side_loops
    assert s.s_f == scaling_factor(1e-3, ps.particle_radius) > 0
    for name in ("predicted_density", "pressure_accel", "verbose", "last_iterations", "last_max_density_error"):
        assert hasattr(s, name), name
    for name in ("compute_densities", "pci_compute_deltas", "pci_scaling_factor", "pci_pos_vel_prediction",
                 "pci_update_pressure", "pci_update_pressure_force", "pci_pc_iteration", "pressure_solve",
                 "compute_pressure_forces", "pci_update_time_step", "substep"):
        assert callable(getattr(s, name)), name
    assert ps._solver_constants()[-1] == 0.0  # no cohesion in the engine parameters


def test_step_is_one_library_call(fake_engine):
    from sph_taichi_b200.PCISPH import scaling_factor
    ps, s = _solver()
    s.initialize()
    eng = RecordingEngine.last
    eng.log.clear()
    s.step()
    assert eng.log == ["pcisph_step:1:0.01:3:1000:4"]
    assert eng.delta == float(np.float32(scaling_factor(1e-3, ps.particle_radius)))
    assert (s.last_iterations, s.last_max_density_error) == (7, 4.5)
    eng.log.clear()
    s.dt[None] = 5e-4  # delta follows the time step
    s.step(3)  # the next first batch is the last step's sweep count
    assert eng.log == ["set_params", "pcisph_step:3:0.01:3:1000:7"]  # the new dt reaches the engine first
    assert eng.delta == float(np.float32(scaling_factor(5e-4, ps.particle_radius)))


@pytest.mark.parametrize("errs, sweeps", [
    ([1.0, 1.0, 1.0, 1.0], 3),                 # at least 3 sweeps even when the first meets eta
    ([50.0, 30.0, 20.0, 10.0, 9.5, 1.0], 5),   # then the first sweep under 1 % rho0 (10.0 itself does not stop it)
])
def test_host_loop_runs_the_legacy_op_sequence(fake_engine, errs, sweeps):
    ps, s = _solver()
    s.device_side_loops = False
    s.initialize()
    eng = RecordingEngine.last
    eng.log.clear()
    RecordingEngine.errs = list(errs)
    s.step()
    assert eng.log == (["neighbor_build", "boundary_volume", "pcisph:0", "pcisph:1"]
                       + ["pcisph:2", "pcisph:3", "pcisph:4"] * sweeps
                       + ["pcisph:5", "pcisph:6", "enforce_boundary"]), eng.log
    assert s.last_iterations == sweeps and s.last_max_density_error == errs[sweeps - 1]


def test_host_loop_stops_at_the_cap(fake_engine):
    ps, s = _solver()
    s.device_side_loops = False
    s.max_iterations = 4
    s.initialize()
    RecordingEngine.errs = [100.0] * 10
    s.step()
    assert s.last_iterations == 4 and len(RecordingEngine.errs) == 6
    s.device_side_loops = True
    eng = RecordingEngine.last
    eng.log.clear()
    s.pressure_solve()  # on its own: the device-side loop
    assert eng.log == ["pcisph_solve:0.01:3:4:4"] and s.last_iterations == 5


def test_sharding_refuses_pcisph_before_any_device_work(monkeypatch):
    from sph_taichi_b200 import engine, slab

    def no_engine(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(engine, "Engine", no_engine)
    with pytest.raises(NotImplementedError, match="not simulationMethod 1"):
        slab.build_sharded(_pcisph_scene(), 0, 1, None)


def test_cli_gpus_refuses_a_pcisph_scene(tmp_path):
    """run_simulation.py --gpus 1 on a PCISPH scene exits non-zero with the message (host-emulated library)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    from tests.test_slab_gloo_dump import _run
    sc = scene.dam_break_box([6, 6, 6], domain_end=[0.4, 0.4, 0.4], start=[0.1, 0.1, 0.1])
    sc["Configuration"]["simulationMethod"] = 1
    (tmp_path / "pcisph.json").write_text(json.dumps(sc))
    res = _run(1, None, ["main", "--", "--scene_file", str(tmp_path / "pcisph.json"), "--gpus", "1", "--frames", "1"],
               cwd=str(tmp_path), check=False)
    assert res.returncode != 0 and "not simulationMethod 1" in res.stderr, res.stdout[-2000:] + res.stderr[-2000:]
    assert not os.path.exists(tmp_path / "pcisph_output")
