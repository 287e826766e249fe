"""Sharded scenes with static solids on the CPU: the host-emulated build of the library over gloo
(``slab.GlooTransport`` stands in for NCCL).  A static rigid block lies under the fluid and across every cut: its
records travel through the send staging unchanged, its start-up boundary volumes are the single engine's, and the
sharded WCSPH and DFSPH runs must reproduce the single engine particle by particle (matched by object_id and x_0).
Dynamic solids are refused at both layers."""
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


def _run(nproc, port, extra, lib=None, env_extra=None):
    import build_emu
    lib = lib or build_emu.build()
    args = [SCRIPT, "--static-block", *extra]
    if nproc == 1:
        cmd = [sys.executable, *args]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
               "127.0.0.1", "--master-port", str(port), *args]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check_static(out):
    assert out["same_particle_set"], out
    assert out["static_solids"] > 0 and out["static_solids_at_x0"], out
    assert out["max_rel_dm_V_static"] < 1e-6, out


def test_static_block_two_ranks_wcsph():
    """Fluid at +3 m/s over the block for 20 steps: particles migrate across the cut, which also cuts the block."""
    out = _run(2, 29581, ["--counts", "24", "8", "8", "--steps", "20", "--vx", "3"])
    _check_static(out)
    assert out["max_dx_over_d"] < 1e-3 and out["max_dv"] < 1e-2, out
    assert out["migrated"], out
    lo, hi = out["solid_layers"]
    assert lo < out["slabs_first"][0][1] < hi, out  # the cut runs through the block
    assert out["ok"], out


def test_static_block_three_ranks_skewed_cuts_rebalanced():
    """Three ranks, every interior cut shifted by two layers and re-balanced every 2 steps (graph replay): the cuts
    move across the block."""
    out = _run(3, 29582, ["--counts", "32", "8", "8", "--steps", "16", "--vx", "3", "--skew", "-2",
                          "--rebalance-every", "2"], env_extra={"SPH_SHARD_GRAPH": "1"})
    _check_static(out)
    assert out["max_dx_over_d"] < 1e-3 and out["max_dv"] < 1e-2, out
    assert out["migrated"] and out["cuts_moved"], out
    lo, hi = out["solid_layers"]
    moved = [(f[1], l_[1]) for f, l_ in zip(out["slabs_first"][:-1], out["slabs_last"][:-1]) if f[1] != l_[1]]
    assert any(lo < a < hi and lo < b < hi for a, b in moved), out
    assert out["ok"], out


def test_static_block_two_ranks_dfsph():
    """DFSPH over the block: the single engine's iteration counts in every step, bit-identical counts and errors on
    every rank, aligned ghosts."""
    out = _run(2, 29583, ["--dfsph", "--counts", "24", "8", "8", "--steps", "20", "--vx", "3"])
    _check_static(out)
    assert out["iterations_sharded"] == out["iterations_single"], out
    assert any(iv + ip > 0 for iv, ip in out["iterations_sharded"]), out  # the Jacobi sweeps (and their exchanges) ran
    assert out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    assert out["max_dx_over_d"] < 2e-3, out
    assert out["migrated"], out
    assert out["ok"], out


def test_dynamic_solids_are_refused():
    """A dynamic rigid block: build_sharded raises for WCSPH and DFSPH; sph_shard_configure refuses a context packed
    with dynamic solids; on a sharded context the calls that would make solids dynamic or walk the solid-id slot map
    are refused.  Every message names the limitation."""
    import build_emu
    lib = build_emu.build()
    code = textwrap.dedent("""
        import ctypes as C, os, sys
        sys.path.insert(0, os.path.join(os.environ["PYTHONPATH"], "tests", "emu"))
        sys.path.insert(0, os.path.join(os.environ["PYTHONPATH"], "tools"))
        import emu_engine
        emu_engine.install(os.environ["SPH_EMU_LIB"])
        import numpy as np, torch
        from sph_taichi_b200 import SimConfig, _lib, engine, scene, slab
        from check_slab_parity import static_block_scene
        cpu = torch.device("cpu")

        def refused(e, rc):
            assert rc != 0 and b"static solids only" in e.lib.sph_last_error(e.ctx), e.lib.sph_last_error(e.ctx)

        for dfsph in (False, True):
            sc = static_block_scene([12, 6, 6], 0.02)
            if dfsph:
                sc = scene._as_dfsph(sc)
            sc["RigidBlocks"][0]["isDynamic"] = True
            try:
                slab.build_sharded(sc, 0, 1, cpu)
                raise SystemExit("build_sharded accepted a dynamic solid")
            except NotImplementedError as exc:
                assert "static solids only" in str(exc), exc
            # the C ABI on its own: a context packed with the dynamic block
            cfg = SimConfig(sc)
            arrays, _, _, counts = scene.assemble_particles(cfg, 3, 0.02)
            arrays["solid_id"] = slab.solid_ids(arrays)
            n, ns = counts["total"], counts["solid"]
            e = engine.Engine(slab.scene_params(cfg), n_max=4 * n, n_solid=ns, n_bodies=1, device=cpu)
            e.set_dfsph(dfsph)
            e.pack(slab.field_tensors(arrays, n, float(np.float32(0.8 * 0.02 ** 3)), cpu), n, ns, True)
            assert e.lib.sph_comm_set_transport(e.ctx, None, 0, 1) == 0
            gx = int(slab.scene_params(cfg).grid_num[0])
            refused(e, e.lib.sph_shard_configure(e.ctx, 0, gx, slab.GHOST_LAYERS, n, 8))
            e.close()
            # a sharded context with the static block: nothing may turn it dynamic or walk its solid ids
            sc["RigidBlocks"][0]["isDynamic"] = False
            sim, _ = slab.build_sharded(sc, 0, 1, cpu)
            e = sim.eng
            refused(e, e.lib.sph_set_solid_count(e.ctx, sim.n_solid, 1))
            refused(e, e.lib.sph_boundary_volume(e.ctx, 1, None))
            refused(e, e.lib.sph_compute_rigid_rest_cm(e.ctx, 0, None))
            body = (_lib.SphRigidBody * 1)()
            body[0].object_id, body[0].solid_begin, body[0].solid_end = 1, 0, 1
            rc = e.lib.sph_set_rigid_bodies(e.ctx, body, 1)
            assert rc != 0, rc
            sim.step(2)  # the context is still usable
            assert sim.info()["owned"] > 0
            e.close()
        print("refused")
    """)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=_env(lib), cwd=ROOT)
    assert res.returncode == 0 and "refused" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def test_static_block_under_address_sanitizer():
    """One world-1 sharded WCSPH run over the block in the ASan build of the emulated library."""
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    lib = build_emu.build(asan=True)
    out = _run(1, None, ["--counts", "12", "6", "6", "--steps", "6", "--vx", "3"], lib=lib,
               env_extra={"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"})
    _check_static(out)
    assert out["ok"], out
