"""Sharded IISPH on the CPU: ``sph_shard_iisph_step`` (ghost alignment, the per-sweep exchanges of a^p and p / rho^2,
the rank-ordered loop check) in the host-emulated build, world_size 1 to 3 over gloo -- ``slab.GlooTransport`` stands
in for NCCL.  The sharded run must keep the single engine's particle set and pressure sweep counts, every rank must
report bit-identical counts and average errors, and after the alignment each ghost record must hold the neighbour's
boundary record of the same position.  Also: the velocity bound, the refusals, and ``run_simulation.py``'s sharded
loop (``--shard-iisph``) against the single-GPU one.

This file is also the launcher of the CLI runs: ``python tests/test_slab_gloo_iisph.py cli ...`` (under
torch.distributed.run for world > 1) with SPH_EMU_LIB pointing at the emulated library."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")
D = 0.02


def _env(lib, extra=None):
    env = dict(os.environ, SPH_EMU_LIB=lib, PYTHONPATH=ROOT, SPH_SHARD_GRAPH="0", SPH_SHARD_SPLIT_DENSITY="0")
    env.pop("SPH_B200_LIB", None)
    env.update(extra or {})
    return env


def _torchrun(nproc, port):
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
            "127.0.0.1", "--master-port", str(port)]


def _run(nproc, port, extra, lib=None, env_extra=None, expect_ok=True):
    import build_emu
    lib = lib or build_emu.build()
    cmd = ([sys.executable] if nproc == 1 else _torchrun(nproc, port)) + [SCRIPT, "--iisph", *extra]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=ROOT)
    if not expect_ok:
        return res
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check(out):
    assert out["same_particle_set"], out
    assert out["iterations_sharded"] == out["iterations_single"], out  # the same sweeps as the single engine
    assert out["max_dx_over_d"] < 2e-3, out  # test_iisph_steps_vs_oracle's bound for matching counts
    assert out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    assert len(set(out["transport_groups"])) == 1, out  # every rank issued the same transport calls
    assert out["ok"], out


def test_sharded_iisph_two_ranks_equal_the_single_engine():
    """Dam break at 3 m/s toward +x for 20 steps, re-balanced every 4: particles cross the cut.  (The whole block moves
    by 1.5 layers, too little to move the cut here; the pressure and three-rank tests below move theirs.)"""
    out = _run(2, 29591, ["--counts", "24", "8", "8", "--steps", "20", "--vx", "3", "--rebalance-every", "4"])
    _check(out)
    assert out["migrated"], out


def test_sharded_iisph_two_ranks_pressure_at_the_cut():
    """Two blocks meet at +-1.5 m/s on the initial cut (--collide): the fluid along the contact plane is compressed
    above rho0, so the acc and aux words the sweeps exchange carry non-zero pressures across the cut.  A build that
    skipped the acc exchange ends this run 4.6e-3 d away from the single engine."""
    out = _run(2, 29592, ["--collide", "--counts", "24", "8", "8", "--steps", "12", "--vx", "1.5"])
    _check(out)
    assert any(e > 0.0 for e in out["avg_err_single"]), out  # the pressure solve did work
    assert out["migrated"] and out["cuts_moved"], out


def test_sharded_iisph_three_ranks_skewed_cuts_rebalanced():
    """Three ranks with every interior cut shifted by two layers, re-balanced on the device every 2 steps."""
    out = _run(3, 29593, ["--counts", "32", "8", "8", "--steps", "14", "--vx", "2", "--skew", "-2",
                          "--rebalance-every", "2"])
    _check(out)
    assert out["migrated"] and out["cuts_moved"], out


def test_sharded_iisph_static_block():
    """Two ranks, the fluid sliding over a static block that spans the cut: every static solid stays exactly at x_0
    with the single engine's start-up m_V."""
    out = _run(2, 29594, ["--static-block", "--counts", "24", "8", "8", "--steps", "10", "--vx", "2"])
    _check(out)
    assert out["static_solids"] > 0 and out["static_solids_at_x0"], out
    assert out["max_rel_dm_V_static"] < 1e-6, out


def test_velocity_bound_flag_raises():
    """|v_x| * dt >= h in one step (45 m/s * 1e-3 s > h = 0.04 m): the advect sets SPH_STATUS_SHARD_VELOCITY and
    ShardedSimulation.info() raises instead of losing the particle silently; 10 m/s stays below the bound."""
    res = _run(1, None, ["--counts", "12", "6", "6", "--steps", "1", "--vx", "45"], expect_ok=False)
    assert res.returncode != 0, res.stdout[-2000:]
    assert "whole cell layer" in res.stderr, res.stderr[-2000:]
    out = _run(1, None, ["--counts", "12", "6", "6", "--steps", "2", "--vx", "10"])
    assert out["ok"], out


def test_sharded_iisph_refusals():
    """The library refuses: the WCSPH and DFSPH sharded steps and the single-GPU IISPH calls on a sharded IISPH context
    (which stays usable and dumps), sph_set_iisph(1) after sph_shard_configure, sph_shard_iisph_step on a DFSPH
    context, and sph_shard_configure_bodies on an IISPH context."""
    import build_emu
    lib = build_emu.build()
    code = textwrap.dedent("""
        import ctypes as C, os, sys
        sys.path.insert(0, os.path.join(os.environ["PYTHONPATH"], "tests", "emu"))
        import emu_engine
        emu_engine.install(os.environ["SPH_EMU_LIB"])
        import numpy as np, torch
        from sph_taichi_b200 import _lib, engine, scene, slab, SimConfig
        cpu = torch.device("cpu")
        def box():
            return scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3)
        def err(e):
            return e.lib.sph_last_error(e.ctx).decode()
        sim, _ = slab.build_sharded(scene._as_iisph(box()), 0, 1, cpu, iisph=True)
        e = sim.eng
        dio = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
        iio = _lib.SphIisphStep(max_iterations=1, omega=0.5, eta=1e-3, n_fluid=1, first_batch=1)
        it, avg = C.c_int32(0), C.c_double(0.0)
        calls = {
            "sph_shard_step": lambda: e.lib.sph_shard_step(e.ctx, 1, None),
            "sph_shard_profile_step": lambda: e.lib.sph_shard_profile_step(e.ctx, (C.c_float * 6)(), None),
            "sph_shard_dfsph_step": lambda: e.lib.sph_shard_dfsph_step(e.ctx, 1, C.byref(dio), None),
            "sph_iisph_step": lambda: e.lib.sph_iisph_step(e.ctx, 1, C.byref(iio), None),
            "sph_iisph_op": lambda: e.lib.sph_iisph_op(e.ctx, 1, 0.0, None, None),
            "sph_iisph_solve": lambda: e.lib.sph_iisph_solve(e.ctx, 1, 0.5, 1e-3, 1, 1, C.byref(it), C.byref(avg), None),
        }
        for name, call in calls.items():
            assert call() != 0, name
            assert "sph_shard_iisph_step" in err(e), (name, err(e))
        assert e.lib.sph_set_iisph(e.ctx, 1) != 0 and "before sph_shard_configure" in err(e), err(e)
        sim.step(2)  # still usable
        assert sim.info()["owned"] == 12 * 6 * 6 and sim.last_iterations >= 1
        assert sim.dump(0)["position"].shape == (12 * 6 * 6, 3)
        e.close()
        # sph_shard_iisph_step on a sharded DFSPH context
        sim, _ = slab.build_sharded(scene._as_dfsph(box()), 0, 1, cpu)
        e = sim.eng
        assert e.lib.sph_shard_iisph_step(e.ctx, 1, C.byref(iio), None) != 0 and "sph_set_iisph(1)" in err(e), err(e)
        e.close()
        # sph_shard_configure_bodies on an IISPH context
        sc = box()
        cfg = SimConfig(sc)
        arrays, _, _, counts = scene.assemble_particles(cfg, 3, 0.02)
        n = counts["total"]
        e = engine.Engine(slab.scene_params(cfg), n_max=4 * n, n_solid=0, n_bodies=1, device=cpu)
        e.pack(slab.field_tensors(arrays, n, float(np.float32(0.8 * 0.02 ** 3)), cpu), n, 0, False)
        e.set_iisph(True)
        rc = e.lib.sph_shard_configure_bodies(e.ctx, 0, int(slab.scene_params(cfg).grid_num[0]), 3, n, 0, None, 0)
        assert rc != 0 and "dynamic solids in IISPH are single-GPU" in err(e), err(e)
        e.close()
        print("refused")
    """)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=_env(lib), cwd=ROOT)
    assert res.returncode == 0 and "refused" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def _body_scene():
    """An IISPH dam break with a dynamic rigid block on its surface."""
    from sph_taichi_b200 import scene
    sc = scene._as_iisph(scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.4, 0.3], start=[0.06] * 3))
    sc["RigidBlocks"] = [{"objectId": 1, "start": [0.1, 0.2, 0.1], "end": [0.15, 0.25, 0.15],
                          "translation": [0.0, 0.0, 0.0], "scale": [1, 1, 1], "velocity": [0.0, 0.0, 0.0],
                          "density": 600.0, "color": [255, 0, 0], "isDynamic": True}]
    return sc


def test_build_sharded_iisph_opt_in_refusals_before_any_device_work(monkeypatch):
    """iisph=True with dynamic solids (in the scene, or dynamic_solids=True) and iisph=True on a scene of another
    solver are refused before any device work."""
    from sph_taichi_b200 import engine, scene, slab

    def no_engine(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(engine, "Engine", no_engine)
    with pytest.raises(NotImplementedError, match="dynamic solids in IISPH scenes are single-GPU"):
        slab.build_sharded(_body_scene(), 0, 1, None, iisph=True)
    with pytest.raises(NotImplementedError, match="dynamic solids in IISPH scenes are single-GPU"):
        slab.build_sharded(_body_scene(), 0, 1, None, iisph=True, dynamic_solids=True)
    sc = scene._as_iisph(scene.dam_break_box([6, 6, 6], domain_end=[0.4, 0.4, 0.4], start=[0.1] * 3))
    with pytest.raises(NotImplementedError, match="dynamic solids in IISPH scenes are single-GPU"):
        slab.build_sharded(sc, 0, 1, None, iisph=True, dynamic_solids=True)
    with pytest.raises(NotImplementedError, match=r"IISPH \(simulationMethod 3\) is single-GPU.*iisph=True"):
        slab.build_sharded(sc, 0, 1, None)
    with pytest.raises(ValueError, match="simulationMethod 4"):
        slab.build_sharded(scene._as_dfsph(sc), 0, 1, None, iisph=True)


def test_cli_shard_iisph_needs_gpus():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "run_simulation.py"), "--scene", "dragon_bath_iisph",
                          "--shard-iisph"], capture_output=True, text=True, timeout=300, cwd=ROOT,
                         env=dict(os.environ, PYTHONPATH=ROOT))
    assert res.returncode != 0 and "--shard-iisph needs --gpus" in res.stderr, res.stderr[-2000:]


# ------------------------------------------------------------------------------------------------------------------
# run_simulation.py's sharded loop with --shard-iisph
# ------------------------------------------------------------------------------------------------------------------
def _export_scene():
    """Two fluid blocks (object 0 is exported) meeting at +-1.5 m/s at the cut of a balanced two-rank start, IISPH,
    exportPly."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from check_slab_parity import colliding_blocks_scene
    from sph_taichi_b200 import scene
    sc = scene._as_iisph(colliding_blocks_scene([24, 6, 6], D, 1.5))
    sc["Configuration"].update(exportPly=True, exportObj=False)
    return sc


def _launch_cli(a):
    """run_simulation.py's loop on a.scene_file in the current directory: run_single, or run_sharded(iisph=True) on
    WORLD_SIZE ranks over gloo (what --gpus N --shard-iisph runs)."""
    sys.path.insert(0, ROOT)
    import emu_engine
    emu_engine.install(os.environ["SPH_EMU_LIB"])
    import torch
    import torch.distributed as dist
    from run_simulation import run_sharded, run_single
    from sph_taichi_b200 import SimConfig, slab
    cfg = SimConfig(a.scene_file)
    name = os.path.basename(a.scene_file).split(".")[0]
    if not a.sharded:
        return run_single(cfg, name, a.frames, quiet=True)
    world = int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        dist.init_process_group("gloo", rank=int(os.environ["RANK"]), world_size=world)
    try:
        return run_sharded(cfg, name, a.frames, torch.device("cpu"),
                           transport=slab.GlooTransport() if world > 1 else None, quiet=True, iisph=True)
    finally:
        if world > 1:
            dist.destroy_process_group()


def test_cli_two_ranks_iisph_ply(tmp_path):
    """run_sharded(iisph=True) on 2 ranks against run_single: 17 steps, exports after render updates 0 and 16
    (output_interval = int(0.016 / 1e-3)); the same files, every frame a one-to-one match within 1e-3 d."""
    import build_emu
    from tests.test_slab_gloo_dump import compare_outputs
    lib = build_emu.build()
    scene_file = tmp_path / "iisph_case.json"
    scene_file.write_text(json.dumps(_export_scene()))
    me = os.path.abspath(__file__)
    args = ["cli", "--scene-file", str(scene_file), "--frames", "17"]
    for nproc, sub, extra in ((1, "single", []), (2, "sharded", ["--sharded"])):
        (tmp_path / sub).mkdir()
        cmd = ([sys.executable] if nproc == 1 else _torchrun(nproc, 29595)) + [me, *args, *extra]
        res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib), cwd=str(tmp_path / sub))
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    names = compare_outputs(str(tmp_path / "single" / "iisph_case_output"), str(tmp_path / "sharded" / "iisph_case_output"), D)
    assert names == ["particle_object_0_000000.ply", "particle_object_0_000001.ply"], names


def test_sharded_iisph_under_address_sanitizer():
    """One world-1 sharded IISPH run of the ASan build of the emulated library."""
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    lib = build_emu.build(asan=True)
    out = _run(1, None, ["--collide", "--counts", "12", "6", "6", "--steps", "6", "--vx", "1.5"], lib=lib,
               env_extra={"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"})
    assert out["ok"] and out["same_particle_set"] and out["iterations_sharded"] == out["iterations_single"], out


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["cli"])
    ap.add_argument("--scene-file", default="")
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--sharded", action="store_true")
    sys.exit(_launch_cli(ap.parse_args()) or 0)
