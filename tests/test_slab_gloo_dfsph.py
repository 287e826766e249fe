"""Sharded DFSPH on the CPU: ``sph_shard_dfsph_step`` (ghost alignment, per-sweep exchanges, rank-ordered convergence
check) in the host-emulated build, world_size 2 and 3 over gloo -- ``slab.GlooTransport`` stands in for NCCL.  The
sharded run must keep the single engine's particle set and Jacobi iteration counts, every rank must report
bit-identical counts and average errors, and after the alignment each ghost record must hold the neighbour's boundary
record of the same position."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")


def _env(lib, extra=None):
    env = dict(os.environ, SPH_EMU_LIB=lib, PYTHONPATH=ROOT, SPH_SHARD_GRAPH="0", SPH_SHARD_SPLIT_DENSITY="0")
    env.pop("SPH_B200_LIB", None)
    env.update(extra or {})
    return env


def _run(nproc, port, extra, lib=None, env_extra=None, expect_ok=True):
    import build_emu
    lib = lib or build_emu.build()
    if nproc == 1:
        cmd = [sys.executable, SCRIPT, "--dfsph", *extra]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
               "127.0.0.1", "--master-port", str(port), SCRIPT, "--dfsph", *extra]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=ROOT)
    if not expect_ok:
        return res
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check(out):
    assert out["same_particle_set"], out
    assert out["iterations_sharded"] == out["iterations_single"], out  # the same sweeps as the single engine
    assert out["max_dx_over_d"] < 2e-3, out  # test_dfsph_steps_vs_oracle's bound for matching counts
    assert out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    assert out["migrated"] and out["cuts_moved"], out
    assert out["ok"], out


def test_sharded_dfsph_two_ranks_equal_the_single_engine():
    """Dam break at 3 m/s toward +x for 20 steps: particles cross the cut every few steps and the cut moves."""
    out = _run(2, 29571, ["--counts", "24", "8", "8", "--steps", "20", "--vx", "3"])
    _check(out)
    assert len(set(out["transport_groups"])) == 1, out  # every rank issued the same transport calls


def test_sharded_dfsph_three_ranks_skewed_cuts_rebalanced():
    """Three ranks with every interior cut shifted by two layers, re-balanced on the device every 2 steps."""
    out = _run(3, 29572, ["--counts", "32", "8", "8", "--steps", "14", "--vx", "2", "--skew", "-2",
                          "--rebalance-every", "2"])
    _check(out)
    assert len(set(out["transport_groups"])) == 1, out


def test_velocity_bound_flag_raises():
    """|v_x| * dt >= h in one step (12 m/s * 4e-3 s > h = 0.04 m): the advect sets SPH_STATUS_SHARD_VELOCITY and
    ShardedSimulation.info() raises instead of losing the particle silently."""
    res = _run(1, None, ["--counts", "12", "6", "6", "--steps", "1", "--vx", "12"], expect_ok=False)
    assert res.returncode != 0, res.stdout[-2000:]
    assert "whole cell layer" in res.stderr, res.stderr[-2000:]
    out = _run(1, None, ["--counts", "12", "6", "6", "--steps", "2", "--vx", "4"])  # below the bound: no flag
    assert out["ok"], out


def test_sharded_entry_points_refuse_the_other_solver():
    """sph_shard_step refuses a DFSPH context, sph_dfsph_step a sharded one, sph_shard_dfsph_step a WCSPH one."""
    import build_emu
    lib = build_emu.build()
    code = textwrap.dedent("""
        import ctypes as C, os, sys
        sys.path.insert(0, os.path.join(os.environ["PYTHONPATH"], "tests", "emu"))
        import emu_engine
        emu_engine.install(os.environ["SPH_EMU_LIB"])
        import torch
        from sph_taichi_b200 import _lib, scene, slab
        for dfsph in (True, False):
            sc = scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3)
            if dfsph:
                sc = scene._as_dfsph(sc)
            sim, _ = slab.build_sharded(sc, 0, 1, torch.device("cpu"))
            e = sim.eng
            io = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
            if dfsph:
                assert e.lib.sph_shard_step(e.ctx, 1, None) != 0
                assert b"sph_shard_dfsph_step" in e.lib.sph_last_error(e.ctx)
                assert e.lib.sph_dfsph_step(e.ctx, 1, C.byref(io), None) != 0
                assert b"sph_shard_dfsph_step" in e.lib.sph_last_error(e.ctx)
            else:
                assert e.lib.sph_shard_dfsph_step(e.ctx, 1, C.byref(io), None) != 0
        print("refused")
    """)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=_env(lib), cwd=ROOT)
    assert res.returncode == 0 and "refused" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def test_sharded_dfsph_under_address_sanitizer():
    """One world-1 sharded DFSPH run of the ASan build of the emulated library."""
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    lib = build_emu.build(asan=True)
    out = _run(1, None, ["--counts", "12", "6", "6", "--steps", "6", "--vx", "3"], lib=lib,
               env_extra={"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"})
    assert out["ok"] and out["same_particle_set"] and out["iterations_sharded"] == out["iterations_single"], out
