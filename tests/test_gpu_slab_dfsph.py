"""Sharded DFSPH (sph_shard_dfsph_step) on the GPU: a world-1 sharded run against the plain DFSPH engine, and two
GPUs over NCCL against one (skipped with fewer than two GPUs)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")


def _run(nproc, extra):
    if nproc == 1:
        cmd = [sys.executable, SCRIPT, "--dfsph", *extra]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", "29573", SCRIPT, "--dfsph", *extra]
    env = dict(os.environ, SPH_SHARD_GRAPH="0")  # SPH_EMU_LIB, if set, routes the tool to the emulated library
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def test_sharded_dfsph_single_rank_equals_plain_engine():
    """World 1: slab classification, trash bucket, owned-range kernels and the rank-ordered check without any
    exchange -- the same iteration counts as sph_dfsph_step in every step and |dx|/d < 1e-4 after 30 steps."""
    out = _run(1, ["--counts", "40", "16", "16", "--steps", "30", "--vx", "2"])
    assert out["same_particle_set"], out
    assert out["iterations_sharded"] == out["iterations_single"], out
    assert out["max_dx_over_d"] < 1e-4, out
    assert out["ok"], out


def test_sharded_dfsph_two_gpus_equal_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _run(2, ["--counts", "64", "24", "24", "--steps", "40", "--vx", "3"])
    assert out["same_particle_set"] and out["bit_identical_across_ranks"] and out["ghosts_aligned"], out
    assert out["migrated"], out
    assert out["ok"], out


def test_sharded_entry_points_refuse_the_other_solver():
    import ctypes as C
    import torch
    from sph_taichi_b200 import _lib, scene, slab
    for dfsph in (True, False):
        sc = scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3)
        if dfsph:
            sc = scene._as_dfsph(sc)
        dev = torch.device("cpu") if os.environ.get("SPH_EMU_LIB") else torch.device("cuda:0")
        sim, _ = slab.build_sharded(sc, 0, 1, dev)
        e = sim.eng
        io = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
        if dfsph:
            assert e.lib.sph_shard_step(e.ctx, 1, e._stream()) != 0
            assert e.lib.sph_dfsph_step(e.ctx, 1, C.byref(io), e._stream()) != 0
            sim.step(2)  # the context is still usable
            sim.synchronize()
            assert sim.info()["owned"] == 12 * 6 * 6
        else:
            assert e.lib.sph_shard_dfsph_step(e.ctx, 1, C.byref(io), e._stream()) != 0
        e.close()
