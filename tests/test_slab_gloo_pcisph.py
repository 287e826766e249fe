"""Sharded PCISPH on the CPU: ``sph_shard_pcisph_step`` (ghost alignment, the per-sweep exchanges of {x*, m_V} and p,
the max of the ranks' error partials) in the host-emulated build, world_size 1 to 3 over gloo -- ``slab.GlooTransport``
stands in for NCCL.  The sharded run must keep the single engine's particle set and sweep counts, every rank must
report bit-identical counts and max errors, and after the alignment each ghost record must hold the neighbour's
boundary record of the same position.  Also: the velocity bound, the refusals, and ``run_simulation.py``'s sharded
loop (``--shard-pcisph``) against the single-GPU one.

This file is also the launcher of the CLI runs: ``python tests/test_slab_gloo_pcisph.py cli ...`` (under
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
    cmd = ([sys.executable] if nproc == 1 else _torchrun(nproc, port)) + [SCRIPT, "--pcisph", *extra]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=ROOT)
    if not expect_ok:
        return res
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check(out):
    assert out["same_particle_set"], out
    assert out["iterations_sharded"] == out["iterations_single"], out  # the same sweeps as the single engine
    assert out["max_dx_over_d"] < 1e-3, out  # test_pcisph_steps_vs_oracle's bound for matching counts
    assert out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    assert len(set(out["transport_groups"])) == 1, out  # every rank issued the same transport calls
    assert out["ok"], out


def test_sharded_pcisph_two_ranks_equal_the_single_engine():
    """Dam break at 3 m/s toward +x for 20 steps, re-balanced every 4: particles cross the cut."""
    out = _run(2, 29691, ["--counts", "24", "8", "8", "--steps", "20", "--vx", "3", "--rebalance-every", "4"])
    _check(out)
    assert out["migrated"], out


def test_sharded_pcisph_two_ranks_pressure_at_the_cut():
    """Two blocks meet at +-3 m/s on the initial cut (--collide): the fluid along the contact plane is compressed above
    rho0, so the predicted positions and the pressures the sweeps exchange act across the cut, and some steps run more
    than the minimum of 3 sweeps.  Measured on scratch builds of the emulated library: without the {x*, m_V} message
    (DX_DFS) the first ghost layer keeps stale predicted positions and a particle reaches |v_x| dt >= h within the run
    (the velocity flag ends it); without the pressure message (DX_MISC, the error all-gather kept) the run ends
    0.159 d from the single engine with different sweep counts.  This build ends 4.5e-6 d from it."""
    out = _run(2, 29692, ["--collide", "--counts", "24", "8", "8", "--steps", "16", "--vx", "3"])
    _check(out)
    assert max(c[0] for c in out["iterations_single"]) > 3, out  # the loop ran past its minimum
    assert any(e > 0.0 for e in out["max_err_single"]), out
    assert out["migrated"], out


def test_sharded_pcisph_three_ranks_skewed_cuts_rebalanced():
    """Three ranks with every interior cut shifted by two layers, re-balanced on the device every 2 steps."""
    out = _run(3, 29693, ["--counts", "32", "8", "8", "--steps", "14", "--vx", "2", "--skew", "-2",
                          "--rebalance-every", "2"])
    _check(out)
    assert out["migrated"] and out["cuts_moved"], out


def test_sharded_pcisph_static_block():
    """Two ranks, the fluid sliding 1.5 spacings above a static block that spans the cut: every static solid stays
    exactly at x_0 with the single engine's start-up m_V.  (One spacing above it, as the IISPH test has it, the fluid's
    bottom layer starts far above rho0 and the single engine's max-error loop runs to its cap: DESIGN section 11.)"""
    out = _run(2, 29694, ["--static-block", "--block-gap", "1.5", "--counts", "24", "8", "8", "--steps", "10",
                          "--vx", "2"])
    _check(out)
    assert max(c[0] for c in out["iterations_single"]) < 10, out  # far below the cap
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


def _body_scene():
    """A PCISPH dam break with a dynamic rigid block on its surface."""
    from sph_taichi_b200 import scene
    sc = scene._as_pcisph(scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.4, 0.3], start=[0.06] * 3))
    sc["RigidBlocks"] = [{"objectId": 1, "start": [0.1, 0.2, 0.1], "end": [0.15, 0.25, 0.15],
                          "translation": [0.0, 0.0, 0.0], "scale": [1, 1, 1], "velocity": [0.0, 0.0, 0.0],
                          "density": 600.0, "color": [255, 0, 0], "isDynamic": True}]
    return sc


def test_build_sharded_pcisph_opt_in_refusals_before_any_device_work(monkeypatch):
    """pcisph=True with dynamic solids (in the scene, or dynamic_solids=True), pcisph=True on a scene of another solver,
    and a PCISPH scene without the opt-in are refused before any device work."""
    from sph_taichi_b200 import engine, scene, slab

    def no_engine(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(engine, "Engine", no_engine)
    sc = scene._as_pcisph(scene.dam_break_box([6, 6, 6], domain_end=[0.4, 0.4, 0.4], start=[0.1] * 3))
    for kw in ({}, {"dynamic_solids": True}):
        with pytest.raises(NotImplementedError) as exc:
            slab.build_sharded(_body_scene(), 0, 1, None, pcisph=True, **kw)
        assert str(exc.value) == slab.DYNAMIC_SOLIDS_PCISPH
    with pytest.raises(NotImplementedError, match="dynamic solids in PCISPH scenes are single-GPU"):
        slab.build_sharded(sc, 0, 1, None, pcisph=True, dynamic_solids=True)
    with pytest.raises(NotImplementedError, match=r"not simulationMethod 1 unless requested.*pcisph=True"):
        slab.build_sharded(sc, 0, 1, None)
    with pytest.raises(NotImplementedError, match="not simulationMethod 1"):
        slab.build_sharded(sc, 0, 1, None, iisph=True)
    with pytest.raises(ValueError, match="iisph=True shards an IISPH scene"):
        slab.build_sharded(sc, 0, 1, None, pcisph=True, iisph=True)
    for as_method, method in ((scene._as_dfsph, 4), (scene._as_iisph, 3), (lambda s: s, 0)):
        other = as_method(scene.dam_break_box([6, 6, 6], domain_end=[0.4, 0.4, 0.4], start=[0.1] * 3))
        assert other["Configuration"]["simulationMethod"] == method
        with pytest.raises(ValueError) as exc:
            slab.build_sharded(other, 0, 1, None, pcisph=True)
        assert str(exc.value) == (f"pcisph=True shards a PCISPH scene (simulationMethod 1), not simulationMethod "
                                  f"{method}")
    assert slab.shard_mode(1, False, pcisph=True) == slab.ShardMode(slab.Solver.PCISPH, False)


def test_sharded_pcisph_refusal_table():
    """The library's refusals around a sharded PCISPH context, configured (sph_shard_configure_pcisph) and begun
    (sph_shard_begin): the single-GPU PCISPH calls and the other solvers' steps name sph_shard_pcisph_step;
    sph_set_pcisph(1) and the other configure calls keep their message; sph_shard_pcisph_step needs sph_shard_begin;
    sph_shard_configure_pcisph refuses the other solvers and dynamic solids; sph_shard_pcisph_step refuses unsharded
    and other solvers' contexts.  The begun context still steps, reports and dumps."""
    import build_emu
    lib = build_emu.build()
    code = textwrap.dedent("""
        import ctypes as C, os, sys
        sys.path.insert(0, os.path.join(os.environ["PYTHONPATH"], "tests", "emu"))
        import emu_engine
        emu_engine.install(os.environ["SPH_EMU_LIB"])
        import numpy as np, torch
        from sph_taichi_b200 import _lib, engine, scene, slab, SimConfig
        from tests.test_slab_gloo_pcisph import _body_scene
        cpu = torch.device("cpu")
        SHARDED = "this PCISPH context is sharded: step it with sph_shard_pcisph_step"
        SHARD_STEP = "this context is in PCISPH mode (sph_set_pcisph): a sharded PCISPH context steps with sph_shard_pcisph_step"
        SINGLE_GPU = "PCISPH (sph_set_pcisph) is single-GPU: x-slab sharding runs WCSPH, DFSPH and IISPH contexts"
        NEEDS_PCISPH = ("sph_shard_configure_pcisph shards a PCISPH context: call sph_set_pcisph(1) before it (WCSPH, "
                        "DFSPH and IISPH contexts use sph_shard_configure)")
        DYNAMIC = "x-slab sharding of a PCISPH context runs fluid and static solids: dynamic solids in PCISPH are single-GPU"
        def box():
            return scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3)
        def err(e):
            return e.lib.sph_last_error(e.ctx).decode()
        def context(sc, solver, dynamic=False):
            cfg = SimConfig(sc)
            arrays, _, _, counts = scene.assemble_particles(cfg, 3, 0.02)
            n = counts["total"]
            n_solid = int((np.asarray(arrays["material"]) != 1).sum())
            if n_solid:
                arrays["solid_id"] = slab.solid_ids(arrays)
            e = engine.Engine(slab.scene_params(cfg), n_max=4 * n, n_solid=n_solid, n_bodies=1, device=cpu)
            e.pack(slab.field_tensors(arrays, n, float(np.float32(0.8 * 0.02 ** 3)), cpu), n, n_solid, dynamic)
            if solver:
                getattr(e, "set_" + solver)(True)
            e._check(e.lib.sph_comm_set_transport(e.ctx, None, 0, 1), "sph_comm_set_transport")
            return e, n, int(slab.scene_params(cfg).grid_num[0])
        def refuses(e, rc, text):
            assert rc != 0 and err(e) == text, (rc, err(e), text)

        dio = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
        iio = _lib.SphIisphStep(max_iterations=1, omega=0.5, eta=1e-3, n_fluid=1, first_batch=1)
        pio = _lib.SphPcisphStep(delta=700.0, eta=0.01, min_iterations=3, max_iterations=10, first_batch=1)
        it, mx = C.c_int32(0), C.c_double(0.0)
        # configured, then begun
        e, n, gx = context(scene._as_pcisph(box()), "pcisph")
        assert e.lib.sph_shard_configure_pcisph(e.ctx, 0, gx, 2, n, 0) == 0, err(e)
        refuses(e, e.lib.sph_shard_pcisph_step(e.ctx, 1, C.byref(pio), None), "sph_shard_begin was not called")
        for begun in (False, True):
            if begun:
                assert e.lib.sph_shard_begin(e.ctx, None) == 0, err(e)
            refuses(e, e.lib.sph_pcisph_step(e.ctx, 1, C.byref(pio), None), SHARDED)
            refuses(e, e.lib.sph_pcisph_op(e.ctx, 1, 0.0, None, None), SHARDED)
            refuses(e, e.lib.sph_pcisph_solve(e.ctx, 700.0, 0.01, 3, 10, 1, C.byref(it), C.byref(mx), None), SHARDED)
            refuses(e, e.lib.sph_shard_step(e.ctx, 1, None), SHARD_STEP)
            refuses(e, e.lib.sph_shard_profile_step(e.ctx, (C.c_float * 6)(), None), SHARD_STEP)
            refuses(e, e.lib.sph_shard_dfsph_step(e.ctx, 1, C.byref(dio), None), SHARD_STEP)
            refuses(e, e.lib.sph_shard_iisph_step(e.ctx, 1, C.byref(iio), None), SHARD_STEP)
            refuses(e, e.lib.sph_set_pcisph(e.ctx, 1), SINGLE_GPU)
            refuses(e, e.lib.sph_shard_configure(e.ctx, 0, gx, 2, n, 0), SINGLE_GPU)
            refuses(e, e.lib.sph_shard_configure_bodies(e.ctx, 0, gx, 3, n, 0, None, 0), SINGLE_GPU)
            refuses(e, e.lib.sph_shard_configure_iisph_bodies(e.ctx, 0, gx, 3, n, 0, None, 0), SINGLE_GPU)
            refuses(e, e.lib.sph_step(e.ctx, 1, None), "this context is in PCISPH mode (sph_set_pcisph): it steps with "
                    "sph_pcisph_op / sph_pcisph_solve / sph_pcisph_step")
        pio.delta = 735.0
        assert e.lib.sph_shard_pcisph_step(e.ctx, 2, C.byref(pio), None) == 0, err(e)
        assert pio.iterations >= 3
        info = (C.c_int32 * 16)()
        assert e.lib.sph_shard_info(e.ctx, info, None, None) == 0 and info[1] == 12 * 6 * 6 and info[14] == 0
        x = torch.zeros((n, 3)); v = torch.zeros((n, 3))
        rows, status = C.c_int64(0), C.c_uint32(0)
        assert e.lib.sph_shard_dump(e.ctx, 0, C.c_void_p(x.data_ptr()), C.c_void_p(v.data_ptr()), n, C.byref(rows),
                                    C.byref(status), None) == 0, err(e)
        assert rows.value == n
        e.close()
        # sph_shard_configure_pcisph on the other solvers' contexts and on a PCISPH context with dynamic solids
        for solver in (None, "dfsph", "iisph"):
            e, n, gx = context(box(), solver)
            refuses(e, e.lib.sph_shard_configure_pcisph(e.ctx, 0, gx, 2, n, 0), NEEDS_PCISPH)
            e.close()
        e, n, gx = context(_body_scene(), "pcisph", dynamic=True)
        refuses(e, e.lib.sph_shard_configure_pcisph(e.ctx, 0, gx, 2, n, 0), DYNAMIC)
        e.close()
        # sph_shard_pcisph_step on an unsharded PCISPH context and on sharded contexts of other solvers
        e, n, gx = context(scene._as_pcisph(box()), "pcisph")
        refuses(e, e.lib.sph_shard_pcisph_step(e.ctx, 1, C.byref(pio), None), "sph_shard_configure was not called")
        e.close()
        for solver, text in ((None, "sph_set_pcisph(1) was not called before sph_shard_configure_pcisph"),
                             ("iisph", "this context is in IISPH mode (sph_set_iisph): a sharded IISPH context steps "
                                       "with sph_shard_iisph_step")):
            e, n, gx = context(box(), solver)
            assert e.lib.sph_shard_configure(e.ctx, 0, gx, 2, n, 0) == 0, err(e)
            assert e.lib.sph_shard_begin(e.ctx, None) == 0, err(e)
            refuses(e, e.lib.sph_shard_pcisph_step(e.ctx, 1, C.byref(pio), None), text)
            e.close()
        print("refused")
    """)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=_env(lib), cwd=ROOT)
    assert res.returncode == 0 and "refused" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def test_cli_shard_pcisph_needs_gpus():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "run_simulation.py"), "--scene", "dragon_bath_pcisph",
                          "--shard-pcisph"], capture_output=True, text=True, timeout=300, cwd=ROOT,
                         env=dict(os.environ, PYTHONPATH=ROOT))
    assert res.returncode != 0 and "--shard-pcisph needs --gpus" in res.stderr, res.stderr[-2000:]


# ------------------------------------------------------------------------------------------------------------------
# run_simulation.py's sharded loop with --shard-pcisph
# ------------------------------------------------------------------------------------------------------------------
def _export_scene():
    """Two fluid blocks (object 0 is exported) meeting at +-1.5 m/s at the cut of a balanced two-rank start, PCISPH,
    exportPly."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from check_slab_parity import colliding_blocks_scene
    from sph_taichi_b200 import scene
    sc = scene._as_pcisph(colliding_blocks_scene([24, 6, 6], D, 1.5))
    sc["Configuration"].update(exportPly=True, exportObj=False)
    return sc


def _launch_cli(a):
    """run_simulation.py's loop on a.scene_file in the current directory: run_single, or run_sharded(pcisph=True) on
    WORLD_SIZE ranks over gloo (what --gpus N --shard-pcisph runs)."""
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
                           transport=slab.GlooTransport() if world > 1 else None, quiet=True, pcisph=True)
    finally:
        if world > 1:
            dist.destroy_process_group()


def test_cli_two_ranks_pcisph_ply(tmp_path):
    """run_sharded(pcisph=True) on 2 ranks against run_single: 17 steps, exports after render updates 0 and 16
    (output_interval = int(0.016 / 1e-3)); the same files, every frame a one-to-one match within 1e-3 d."""
    import build_emu
    from tests.test_slab_gloo_dump import compare_outputs
    lib = build_emu.build()
    scene_file = tmp_path / "pcisph_case.json"
    scene_file.write_text(json.dumps(_export_scene()))
    me = os.path.abspath(__file__)
    args = ["cli", "--scene-file", str(scene_file), "--frames", "17"]
    for nproc, sub, extra in ((1, "single", []), (2, "sharded", ["--sharded"])):
        (tmp_path / sub).mkdir()
        cmd = ([sys.executable] if nproc == 1 else _torchrun(nproc, 29695)) + [me, *args, *extra]
        res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib), cwd=str(tmp_path / sub))
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    names = compare_outputs(str(tmp_path / "single" / "pcisph_case_output"),
                            str(tmp_path / "sharded" / "pcisph_case_output"), D)
    assert names == ["particle_object_0_000000.ply", "particle_object_0_000001.ply"], names


def test_sharded_pcisph_under_address_sanitizer():
    """One world-1 sharded PCISPH run of the ASan build of the emulated library."""
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
