"""Sharded WCSPH scenes with DYNAMIC solids on the CPU: the host-emulated build of the library over gloo
(``slab.GlooTransport`` stands in for NCCL), through ``tools/check_slab_parity.py --dynamic-body --dynamic-block``.
A shape-matched cube straddles the initial cut and rests on the fluid surface; an advected dynamic rigid block rests on
the surface further along.  The sharded run must reproduce the single engine particle by particle (matched by
object_id and x_0), with the body's cm and R bit-identical on every rank after every step."""
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
    args = [SCRIPT, "--dynamic-body", "--dynamic-block", *extra]
    if nproc == 1:
        cmd = [sys.executable, *args]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
               "127.0.0.1", "--master-port", str(port), *args]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check_dynamic(out):
    assert out["same_particle_set"], out
    assert out["dynamic_solids"] > 0 and out["n_bodies"] == 1, out
    assert out["max_dx_over_d_fluid"] < 1e-3 and out["max_dx_over_d"] < 1e-3 and out["max_dv"] < 1e-2, out
    assert out["bodies_bit_identical_across_ranks"], out
    assert out["reactions_acted"], out  # every dynamic object left free fall, in both engines
    assert all(b["dcm_over_d"] < 1e-3 and b["max_dR"] < 1e-3 for b in out["bodies"]), out
    assert out["ok"], out


def test_dynamic_solids_two_ranks():
    """Fluid at +3 m/s under the cube (across the cut) and the block for 20 steps: particles migrate, the cut runs
    through the body, and the body solve adds one transport group per step."""
    out = _run(2, 29591, ["--counts", "24", "8", "8", "--steps", "20", "--vx", "3"])
    _check_dynamic(out)
    assert out["migrated"], out
    body = [b for b in out["bodies"]][0]
    assert body["object_id"] == 2, out
    lo, hi = out["body_layers"]
    assert lo < out["slabs_first"][0][1] < hi, out  # the cut runs through the body
    # per step: the record exchange + the body all-gather; sph_shard_begin: one record exchange
    assert out["transport_groups"] == [1 + 2 * 20] * 2, out


def test_dynamic_solids_three_ranks_skewed_cuts_rebalanced():
    """Three ranks, every interior cut shifted by two layers and re-balanced every 2 steps: a cut moves across the
    body while it is solved across ranks."""
    out = _run(3, 29592, ["--counts", "32", "8", "8", "--steps", "16", "--vx", "3", "--skew", "-2",
                          "--rebalance-every", "2"])
    _check_dynamic(out)
    assert out["migrated"] and out["cuts_moved"], out
    lo, hi = out["body_layers"]
    moved = [(f[1], l_[1]) for f, l_ in zip(out["slabs_first"][:-1], out["slabs_last"][:-1]) if f[1] != l_[1]]
    assert any(lo <= a <= hi or lo <= b <= hi for a, b in moved), out


def test_body_all_gather_bytes():
    """transport_stats, exactly: 4 steps after sph_shard_begin are 5 record exchanges (none feeds a re-balancing step,
    so each carries the narrow send range: 4 record arrays of narrow_cap x 16 bytes + a 64-byte header to the one
    neighbour) and 4 body all-gathers of (world - 1) x body particles x 32 bytes."""
    out = _run(2, 29593, ["--counts", "24", "8", "8", "--steps", "4", "--vx", "3"])
    assert out["ok"], out
    assert out["transport_groups"] == [1 + 2 * 4] * 2, out
    g = 3  # slab.GHOST_LAYERS_BODIES
    for sent, halo_cap in zip(out["transport_bytes"], out["halo_cap"]):
        narrow_cap = (halo_cap * (g + 1) + g + 1) // (g + 2)
        records = 5 * (4 * narrow_cap * 16 + 64)
        bodies = 4 * (2 - 1) * out["body_particles"] * 32
        assert sent == records + bodies, (sent, records, bodies, out)


def test_dynamic_solids_under_address_sanitizer():
    """One world-1 sharded run with the cube and the block in the ASan build of the emulated library."""
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    lib = build_emu.build(asan=True)
    out = _run(1, None, ["--counts", "12", "6", "6", "--steps", "6", "--vx", "3"], lib=lib,
               env_extra={"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"})
    assert out["same_particle_set"] and out["max_dx_over_d"] < 1e-3 and out["ok"], out


def test_refusals_of_the_body_entry_points():
    """DFSPH with dynamic solids (Python and C), ghost_layers < 3, and sph_shard_profile_step / sph_set_rigid_bodies on
    a body context are refused; every message names the limitation."""
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
        from check_slab_parity import add_dynamic_solids
        cpu = torch.device("cpu")
        d, c = 0.02, [12, 6, 6]

        def dyn_scene():
            sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * d + 0.2, c[1] * d + 0.4, c[2] * d + 0.12], start=[0.06] * 3)
            return add_dynamic_solids(sc, c, d, 1, True, True)

        # Python: DFSPH with dynamic solids
        try:
            slab.build_sharded(scene._as_dfsph(dyn_scene()), 0, 1, cpu, dynamic_solids=True)
            raise SystemExit("build_sharded accepted DFSPH with dynamic solids")
        except NotImplementedError as exc:
            assert "WCSPH only" in str(exc), exc

        def packed(dfsph):
            cfg = SimConfig(dyn_scene())
            arrays, _, _, counts = scene.assemble_particles(cfg, 3, d)
            arrays["solid_id"] = slab.solid_ids(arrays)
            n, ns = counts["total"], counts["solid"]
            e = engine.Engine(slab.scene_params(cfg), n_max=4 * n, n_solid=ns, n_bodies=1, device=cpu)
            e.set_dfsph(dfsph)
            e.pack(slab.field_tensors(arrays, n, float(np.float32(0.8 * d ** 3)), cpu), n, ns, True)
            assert e.lib.sph_comm_set_transport(e.ctx, None, 0, 1) == 0
            body = (_lib.SphRigidBody * 1)()
            b = slab.dynamic_bodies(cfg, arrays)[0]
            body[0].object_id, body[0].solid_begin, body[0].solid_end = b
            body[0].rest_cm = (C.c_float * 3)(0.3, 0.3, 0.15)
            return e, int(slab.scene_params(cfg).grid_num[0]), n, body

        def refused(e, rc, what):
            msg = e.lib.sph_last_error(e.ctx)
            assert rc != 0 and what in msg, msg

        # C: DFSPH context, ghost_layers < 3
        e, gx, n, body = packed(True)
        refused(e, e.lib.sph_shard_configure_bodies(e.ctx, 0, gx, 3, n, 8, body, 1), b"WCSPH only")
        e.close()
        e, gx, n, body = packed(False)
        refused(e, e.lib.sph_shard_configure_bodies(e.ctx, 0, gx, 2, n, 8, body, 1), b"ghost_layers >= 3")
        # a body context: stepping works; the timing step, a new body table and the per-body calls are refused
        assert e.lib.sph_shard_configure_bodies(e.ctx, 0, gx, 3, n, 8, body, 1) == 0, e.lib.sph_last_error(e.ctx)
        assert e.lib.sph_shard_begin(e.ctx, None) == 0
        assert e.lib.sph_shard_step(e.ctx, 2, None) == 0, e.lib.sph_last_error(e.ctx)
        buf = (C.c_float * 6)()
        refused(e, e.lib.sph_shard_profile_step(e.ctx, buf, None), b"sph_shard_configure_bodies")
        refused(e, e.lib.sph_set_rigid_bodies(e.ctx, body, 1), b"static solids only")
        refused(e, e.lib.sph_set_rigid_bodies(e.ctx, body, 0), b"fixed")
        refused(e, e.lib.sph_boundary_volume(e.ctx, 1, None), b"static solids only")
        refused(e, e.lib.sph_compute_rigid_rest_cm(e.ctx, 0, None), b"static solids only")
        R, cm = e.rigid_state(0)  # allowed: every rank holds the same cm and R
        assert np.isfinite(cm).all() and abs(np.linalg.det(R) - 1.0) < 1e-4, (R, cm)
        e.close()
        print("refused")
    """)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=_env(lib), cwd=ROOT)
    assert res.returncode == 0 and "refused" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
