"""Sharded PCISPH (sph_shard_pcisph_step) on the GPU: world-1 sharded runs against the plain PCISPH engine,
dragon_bath_pcisph at full size, two GPUs over NCCL against one (skipped with fewer than two GPUs), and the refusals on a
CUDA context."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")


def _run(nproc, extra, timeout=900):
    if nproc == 1:
        cmd = [sys.executable, SCRIPT, "--pcisph", *extra]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", "29584", SCRIPT, "--pcisph", *extra]
    env = dict(os.environ, SPH_SHARD_GRAPH="0")  # SPH_EMU_LIB, if set, routes the tool to the emulated library
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def test_sharded_pcisph_single_rank_equals_plain_engine():
    """World 1: slab classification, trash bucket, owned-range kernels and the ranked max without any exchange -- the
    same sweep counts as sph_pcisph_step in every step and |dx|/d < 1e-4 after 30 steps."""
    out = _run(1, ["--counts", "40", "16", "16", "--steps", "30", "--vx", "2"])
    assert out["same_particle_set"], out
    assert out["iterations_sharded"] == out["iterations_single"], out
    assert out["max_dx_over_d"] < 1e-4, out
    assert out["ok"], out


def test_sharded_pcisph_single_rank_with_pressure_equals_plain_engine():
    """The same at world 1 on two blocks that collide at +-2 m/s (--collide): the fluid is compressed above rho0 along
    the contact plane, so the pressures are non-zero."""
    out = _run(1, ["--collide", "--counts", "40", "16", "16", "--steps", "30", "--vx", "2"])
    assert out["same_particle_set"], out
    assert max(out["max_err_single"]) > 0.0, out  # the loop corrected a compression
    assert out["iterations_sharded"] == out["iterations_single"], out
    assert out["max_dx_over_d"] < 1e-4, out
    assert out["ok"], out


def test_sharded_pcisph_full_size_dragon_bath():
    """dragon_bath_pcisph (442 K particles) at world 1 against the plain engine for 150 steps (0.15 s: through the
    block's impact on the bath): the same particle set, a finite state inside the domain, the rule of
    test_pcisph_steps_vs_oracle (|dx|/d < 1e-3 with matching sweep counts, 5e-2 otherwise), every loop ended below its
    cap with its max error under 1 % rho0 (10 kg/m^3)."""
    out = _run(1, ["--scene", "dragon_bath_pcisph", "--steps", "150"], timeout=1500)
    assert out["same_particle_set"] and out["finite_inside_domain"], out
    assert out["max_dx_over_d"] < (1e-3 if out["counts_match"] else 5e-2), out
    assert max(c[0] for c in out["iterations_sharded"]) < 1000, out
    assert max(out["max_err_sharded"]) < 10.0, out
    assert out["ok"], out


def test_sharded_pcisph_two_gpus_equal_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _run(2, ["--collide", "--counts", "64", "24", "24", "--steps", "40", "--vx", "2"])
    assert out["same_particle_set"] and out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    assert out["migrated"], out
    assert out["ok"], out


def test_sharded_pcisph_refusals_on_a_cuda_context():
    """The single-GPU PCISPH calls and the other solvers' sharded steps refuse a sharded PCISPH context, which stays
    usable; sph_set_pcisph(1) is refused on it with its existing message."""
    import ctypes as C

    import torch
    from sph_taichi_b200 import _lib, scene, slab
    sc = scene._as_pcisph(scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3))
    dev = torch.device("cpu") if os.environ.get("SPH_EMU_LIB") else torch.device("cuda:0")
    sim, _ = slab.build_sharded(sc, 0, 1, dev, pcisph=True)
    e = sim.eng
    st = e._stream()
    dio = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
    iio = _lib.SphIisphStep(max_iterations=1, omega=0.5, eta=1e-3, n_fluid=1, first_batch=1)
    pio = _lib.SphPcisphStep(delta=700.0, eta=0.01, min_iterations=3, max_iterations=10, first_batch=1)
    it, err = C.c_int32(0), C.c_double(0.0)
    calls = {
        "sph_shard_step": lambda: e.lib.sph_shard_step(e.ctx, 1, st),
        "sph_shard_profile_step": lambda: e.lib.sph_shard_profile_step(e.ctx, (C.c_float * 6)(), st),
        "sph_shard_dfsph_step": lambda: e.lib.sph_shard_dfsph_step(e.ctx, 1, C.byref(dio), st),
        "sph_shard_iisph_step": lambda: e.lib.sph_shard_iisph_step(e.ctx, 1, C.byref(iio), st),
        "sph_pcisph_step": lambda: e.lib.sph_pcisph_step(e.ctx, 1, C.byref(pio), st),
        "sph_pcisph_op": lambda: e.lib.sph_pcisph_op(e.ctx, 1, 0.0, None, st),
        "sph_pcisph_solve": lambda: e.lib.sph_pcisph_solve(e.ctx, 700.0, 0.01, 3, 10, 1, C.byref(it), C.byref(err), st),
    }
    for name, call in calls.items():
        assert call() != 0, name
        assert b"sph_shard_pcisph_step" in e.lib.sph_last_error(e.ctx), (name, e.lib.sph_last_error(e.ctx))
    assert e.lib.sph_set_pcisph(e.ctx, 1) != 0
    assert b"PCISPH (sph_set_pcisph) is single-GPU" in e.lib.sph_last_error(e.ctx)
    sim.step(2)  # the context is still usable
    sim.synchronize()
    assert sim.info()["owned"] == 12 * 6 * 6 and sim.last_iterations >= 3
    assert sim.dump(0)["position"].shape == (12 * 6 * 6, 3)
    e.close()
