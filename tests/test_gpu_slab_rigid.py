"""Sharded scenes with static solids on the GPU: world-1 sharded runs of the full-size dragon_bath (WCSPH) and
dragon_bath_dfsph against the plain engine, the static-block scene of tools/check_slab_parity.py, and two GPUs over
NCCL against one (skipped with fewer than two GPUs)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")


def _run(nproc, extra, port=29591):
    if nproc == 1:
        cmd = [sys.executable, SCRIPT, *extra]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), SCRIPT, *extra]
    env = dict(os.environ, SPH_SHARD_GRAPH="0")  # SPH_EMU_LIB, if set, routes the tool to the emulated library
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check_static(out):
    assert out["same_particle_set"], out
    assert out["static_solids"] > 0 and out["static_solids_at_x0"], out
    assert out["max_rel_dm_V_static"] < 1e-6, out


def test_dragon_bath_single_rank_equals_plain_engine():
    """World 1, the whole dragon_bath (423 500 fluid + the static dragon) for 20 WCSPH steps."""
    out = _run(1, ["--scene", "dragon_bath", "--steps", "20"])
    _check_static(out)
    assert out["max_dx_over_d"] < 1e-3 and out["max_dv"] < 1e-2, out
    assert out["ok"], out


def test_dragon_bath_dfsph_single_rank_equals_plain_engine():
    """World 1, dragon_bath_dfsph for 18 steps: the fluid hits the floor at step 13 and both Jacobi loops iterate
    from step 14 (divergence) and 17 (pressure); the plain engine's counts in every step.  (From step 19 the splash
    moves particles more than a cell layer in x per step at dt = 4e-3, which sharded DFSPH flags and refuses.)"""
    out = _run(1, ["--scene", "dragon_bath_dfsph", "--dfsph", "--steps", "18"])
    _check_static(out)
    assert out["iterations_sharded"] == out["iterations_single"], out
    assert any(iv + ip > 0 for iv, ip in out["iterations_sharded"]), out
    assert out["max_dx_over_d"] < 2e-3, out
    assert out["ok"], out


def test_static_block_single_rank_wcsph_and_dfsph():
    for extra in ([], ["--dfsph"]):
        out = _run(1, ["--static-block", "--counts", "40", "16", "16", "--steps", "20", "--vx", "3", *extra])
        _check_static(out)
        assert out["max_dx_over_d"] < (2e-3 if extra else 1e-3), out
        assert out["ok"], out


def test_two_gpus_static_solids_equal_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _run(2, ["--static-block", "--counts", "64", "24", "24", "--steps", "40", "--vx", "3"], port=29592)
    _check_static(out)
    _check_cut_through_solids(out)
    assert out["migrated"] and out["ok"], out
    # the balanced dragon_bath cut runs through the fluid, far from the dragon: skew it into the dragon, so that its
    # records sit in the send ranges and are staged and exchanged every step
    out = _run(2, ["--scene", "dragon_bath", "--steps", "20", "--skew", str(_dragon_skew())], port=29593)
    _check_static(out)
    _check_cut_through_solids(out)
    assert out["ok"], out


def _check_cut_through_solids(out):
    lo, hi = out["solid_layers"]
    for slabs in (out["slabs_first"], out["slabs_last"]):
        assert lo < slabs[0][1] < hi, out


def _dragon_skew():
    """Layers between the balanced 2-rank cut of dragon_bath and the middle of the dragon."""
    import numpy as np
    from sph_taichi_b200 import SimConfig, scene, slab
    cfg = SimConfig(scene.dragon_bath())
    arrays, _, _, _ = scene.assemble_particles(cfg, 3, 0.02)
    lay = slab.layer_of(arrays["x"], 0.04)
    gx = int(np.ceil(np.array(cfg.get_cfg("domainEnd")) / 0.04).astype(int)[0])
    cut = slab.plan_slabs(np.bincount(lay, minlength=gx)[:gx], 2)[0][1]
    solid = lay[arrays["material"] == 0]
    return (int(solid.min()) + int(solid.max()) + 1) // 2 - cut
