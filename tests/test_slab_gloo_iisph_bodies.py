"""Sharded IISPH scenes with DYNAMIC solids on the CPU (``build_sharded(iisph_bodies=True)``,
``sph_shard_configure_iisph_bodies``): the host-emulated build of the library over gloo (``slab.GlooTransport`` stands
in for NCCL), through ``tools/check_slab_parity.py --iisph --dynamic-body --dynamic-block``.  A shape-matched cube
straddles the initial cut on the fluid surface and an advected dynamic rigid block rests on the surface further along.
The sharded run must reproduce the single engine particle by particle (matched by object_id and x_0) with its sweep
count in every step, the counts and average errors bit-identical on every rank, and the body's cm and R bit-identical
on every rank after every step.  Also: the transport groups and bytes of a step, the unchanged traffic of a static
IISPH scene, the refusals, and ``run_simulation.py``'s sharded loop (``--shard-iisph-bodies``) against the single-GPU
one.

This file is also the launcher of the CLI runs: ``python tests/test_slab_gloo_iisph_bodies.py cli ...`` (under
torch.distributed.run for world > 1) with SPH_EMU_LIB pointing at the emulated library."""
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
SCRIPT = os.path.join(ROOT, "tools", "check_slab_parity.py")
D = 0.02
G = 3  # slab.GHOST_LAYERS_BODIES
FIRST_BATCH = 4  # IISPH.FIRST_BATCH: sweeps launched before the first wait of the first step


def _env(lib, extra=None):
    env = dict(os.environ, SPH_EMU_LIB=lib, PYTHONPATH=ROOT, SPH_SHARD_GRAPH="0", SPH_SHARD_SPLIT_DENSITY="0")
    env.pop("SPH_B200_LIB", None)
    env.update(extra or {})
    return env


def _torchrun(nproc, port):
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
            "127.0.0.1", "--master-port", str(port)]


def _run(nproc, port, extra, lib=None, env_extra=None, dynamic=True):
    import build_emu
    lib = lib or build_emu.build()
    args = [SCRIPT, "--iisph", *(["--dynamic-body", "--dynamic-block"] if dynamic else []), *extra]
    cmd = ([sys.executable] if nproc == 1 else _torchrun(nproc, port)) + args
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check(out):
    assert out["same_particle_set"], out
    assert out["dynamic_solids"] > 0 and out["n_bodies"] == 1, out
    assert out["iterations_sharded"] == out["iterations_single"], out  # the single engine's sweeps in every step
    assert out["bit_identical_across_ranks"] and out["ghosts_aligned"], out  # counts, errors, body states; alignment
    assert out["max_dx_over_d_fluid"] < 1e-3 and out["max_dx_over_d"] < 1e-3 and out["max_dv"] < 1e-2, out
    assert out["bodies_bit_identical_across_ranks"], out
    assert out["reactions_acted"], out  # every dynamic object left free fall, in both engines
    assert all(b["dcm_over_d"] < 1e-3 and b["max_dR"] < 1e-3 for b in out["bodies"]), out
    assert len(set(out["transport_groups"])) == 1, out  # every rank issued the same transport calls
    assert out["status"] == [0] * out["world"], out
    assert out["ok"], out


def _sweeps_launched(iterations):
    """Sweeps launched per step (device_loop): a first batch of the previous step's count (FIRST_BATCH in the first
    step), then pairs until the loop has ended; the sweeps behind the converged one still issue their transport
    groups."""
    out, batch = [], FIRST_BATCH
    for (it,) in iterations:
        n = batch
        while n < it:
            n += 2
        out.append(n)
        batch = max(1, it)
    return out


def test_iisph_dynamic_solids_two_ranks():
    """Fluid at +3 m/s under the cube (across the cut) and the block for 20 steps: particles migrate and the cut runs
    through the body.

    Also transport_stats, exactly.  Groups: sph_shard_begin's record exchange, then per step the alignment, v*, the
    warm-start aux, two per sweep launched, the final pressures, the body all-gather and the record exchange.  Bytes to
    the one neighbour: an alignment is 4 record arrays of align_cap x 16 bytes + a 16-byte header; v*, aux, acc and the
    final pressures are sweep_cap x 16 bytes each; a sweep's second message also carries the 8-byte error partial; the
    body all-gather is body particles x 32 bytes; a record exchange is 4 arrays of narrow_cap x 16 bytes + a 64-byte
    header, or of halo_cap records when it feeds a re-balancing step (every 8th: the exchanges of steps 7 and 15)."""
    steps = 20
    out = _run(2, 29667, ["--counts", "24", "8", "8", "--steps", str(steps), "--vx", "3"])
    _check(out)
    assert out["migrated"], out
    assert [b["object_id"] for b in out["bodies"]] == [2], out
    lo, hi = out["body_layers"]
    assert lo < out["slabs_first"][0][1] < hi, out  # the cut runs through the body
    sweeps = sum(_sweeps_launched(out["iterations_sharded"]))
    assert out["transport_groups"] == [1 + 6 * steps + 2 * sweeps] * 2, (out, sweeps)
    wide = sum(1 for s_ in range(1, steps + 1) if (s_ + 1) % 8 == 0)
    for sent, halo_cap in zip(out["transport_bytes"], out["halo_cap"]):
        narrow_cap = (halo_cap * (G + 1) + G + 1) // (G + 2)
        align_cap = (halo_cap * G + G + 1) // (G + 2)
        sweep_cap = (halo_cap + G + 1) // (G + 2)
        records = (steps + 1 - wide) * (4 * narrow_cap * 16 + 64) + wide * (4 * halo_cap * 16 + 64)
        per_step = (4 * align_cap * 16 + 16) + 3 * sweep_cap * 16 + out["body_particles"] * 32
        in_sweeps = sweeps * (2 * sweep_cap * 16 + 8)
        assert sent == records + steps * per_step + in_sweeps, (sent, records, per_step, in_sweeps, out)


def test_iisph_dynamic_solids_three_ranks_skewed_cuts_rebalanced():
    """Three ranks, every interior cut shifted by two layers and re-balanced every 2 steps: a cut moves across the
    body while it is solved across ranks."""
    out = _run(3, 29662, ["--counts", "32", "8", "8", "--steps", "16", "--vx", "3", "--skew", "-2",
                          "--rebalance-every", "2"])
    _check(out)
    assert out["migrated"] and out["cuts_moved"], out
    lo, hi = out["body_layers"]
    moved = [(f[1], l_[1]) for f, l_ in zip(out["slabs_first"][:-1], out["slabs_last"][:-1]) if f[1] != l_[1]]
    assert any(lo <= a <= hi or lo <= b <= hi for a, b in moved), out


def test_iisph_dynamic_solids_pressure_at_the_cut():
    """The cube (across the cut) and the block thrown into the resting fluid at -2 m/s (--body-vy): the fluid under
    them is compressed above rho0 within a few steps, so the reactions gathered at the cut carry non-zero pressures,
    p itself included (the mirrored-boundary term reads misc.y of ghost fluid).  A build that skipped the
    final-pressure message (DX_MISC) ends this run 2.1e-2 d away from the single engine (the body's cm 1.9e-2 d)."""
    out = _run(2, 29663, ["--counts", "24", "8", "8", "--steps", "12", "--vx", "0", "--body-vy", "-2"])
    _check(out)
    assert any(e > 0.0 for e in out["avg_err_single"]), out  # the pressure solve did work
    lo, hi = out["body_layers"]
    assert lo < out["slabs_first"][0][1] < hi, out
    # the cube decelerated against the fluid: far from the free fall of a body thrown at -2 m/s
    assert out["dynamic_vy_sharded"]["2"] > out["free_fall_vy"] + 1.0, out


def test_static_iisph_scene_keeps_its_transport_groups_and_bytes():
    """A sharded IISPH scene with fluid and a static block (sph_shard_configure) issues what it issued before dynamic
    solids could be sharded -- the final-pressure message belongs to body contexts only: 65 groups and 1 418 880 bytes
    per rank for these 6 steps on 2 ranks, recorded from the library before this entry point existed."""
    out = _run(2, 29665, ["--static-block", "--counts", "24", "8", "8", "--steps", "6", "--vx", "2"], dynamic=False)
    assert out["ok"] and out["static_solids"] > 0, out
    assert out["iterations_sharded"] == [[6], [1], [1], [2], [2], [1]], out
    assert out["transport_groups"] == [65, 65] and out["transport_bytes"] == [1418880, 1418880], out


def test_gpu_tests_of_the_body_context_on_the_emulated_build():
    """tests/test_gpu_slab_iisph_bodies.py against the host-emulated library: the reaction gather against the plain
    engine's scatter, and the refusals of the new entry point and of a context it configured (its world-1 run of the
    tool is what the sanitizer test below runs at a smaller size)."""
    import build_emu
    lib = build_emu.build()
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "-k",
           "gather or refusals", os.path.join(ROOT, "tests", "test_gpu_slab_iisph_bodies.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib), cwd=ROOT)
    tail = res.stdout[-3000:] + res.stderr[-3000:]
    assert res.returncode == 0, tail
    m = re.search(r"(\d+) passed", res.stdout)
    assert m and int(m.group(1)) == 2 and "skipped" not in res.stdout.splitlines()[-1], tail


def _body_scene():
    """An IISPH dam break with a dynamic rigid block on its surface."""
    from sph_taichi_b200 import scene
    sc = scene._as_iisph(scene.dam_break_box([12, 6, 6], domain_end=[0.6, 0.4, 0.3], start=[0.06] * 3))
    sc["RigidBlocks"] = [{"objectId": 1, "start": [0.1, 0.2, 0.1], "end": [0.15, 0.25, 0.15],
                          "translation": [0.0, 0.0, 0.0], "scale": [1, 1, 1], "velocity": [0.0, 0.0, 0.0],
                          "density": 600.0, "color": [255, 0, 0], "isDynamic": True}]
    return sc


def test_iisph_bodies_on_another_solver_is_refused_before_any_device_work(monkeypatch):
    """iisph_bodies=True on a WCSPH or DFSPH scene is a ValueError before any device work; iisph=True alone on the
    IISPH scene with the dynamic block keeps its refusal, which now names the opt-in."""
    from sph_taichi_b200 import engine, scene, slab

    def no_engine(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(engine, "Engine", no_engine)
    wcsph = _body_scene()
    wcsph["Configuration"]["simulationMethod"] = 0
    with pytest.raises(ValueError, match="iisph_bodies=True shards an IISPH scene.*simulationMethod 0"):
        slab.build_sharded(wcsph, 0, 1, None, iisph_bodies=True)
    with pytest.raises(ValueError, match="simulationMethod 4"):
        slab.build_sharded(scene._as_dfsph(_body_scene()), 0, 1, None, iisph_bodies=True)
    with pytest.raises(NotImplementedError, match=r"single-GPU unless requested: build_sharded\(\.\.\., iisph_bodies=True\)"
                                                  r".*--shard-iisph-bodies"):
        slab.build_sharded(_body_scene(), 0, 1, None, iisph=True)


def test_cli_shard_iisph_bodies_needs_gpus():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "run_simulation.py"), "--scene", "dragon_bath_iisph",
                          "--shard-iisph-bodies"], capture_output=True, text=True, timeout=300, cwd=ROOT,
                         env=dict(os.environ, PYTHONPATH=ROOT))
    assert res.returncode != 0 and "--shard-iisph-bodies needs --gpus" in res.stderr, res.stderr[-2000:]


# ------------------------------------------------------------------------------------------------------------------
# run_simulation.py's sharded loop with --shard-iisph-bodies
# ------------------------------------------------------------------------------------------------------------------
def _export_scene():
    """The dam break (16 x 8 x 8) at rest with the shape-matched cube on its surface across the cut of a balanced
    two-rank start, IISPH, exportPly + exportObj."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from check_slab_parity import add_dynamic_solids
    from sph_taichi_b200 import scene
    c = [16, 8, 8]
    sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * D + 0.2, c[1] * D + 0.4, c[2] * D + 0.12], start=[0.06] * 3)
    sc = scene._as_iisph(add_dynamic_solids(sc, c, D, 2, True, False))
    sc["Configuration"].update(exportPly=True, exportObj=True)
    return sc


def _launch_cli(a):
    """run_simulation.py's loop on a.scene_file in the current directory: run_single, or
    run_sharded(iisph_bodies=True) on WORLD_SIZE ranks over gloo (what --gpus N --shard-iisph-bodies runs)."""
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
                           transport=slab.GlooTransport() if world > 1 else None, quiet=True, iisph_bodies=True)
    finally:
        if world > 1:
            dist.destroy_process_group()


def test_cli_two_ranks_iisph_bodies_ply_and_obj(tmp_path):
    """run_sharded(iisph_bodies=True) on 2 ranks against run_single, the cube across the cut: 17 steps, exports after
    render updates 0 and 16 (output_interval = int(0.016 / 1e-3)); the same files, every PLY frame a one-to-one match
    and every posed OBJ vertex within 1e-3 d."""
    import build_emu
    from tests.test_slab_gloo_dump import compare_outputs
    lib = build_emu.build()
    scene_file = tmp_path / "iisph_body_case.json"
    scene_file.write_text(json.dumps(_export_scene()))
    me = os.path.abspath(__file__)
    args = ["cli", "--scene-file", str(scene_file), "--frames", "17"]
    for nproc, sub, extra in ((1, "single", []), (2, "sharded", ["--sharded"])):
        (tmp_path / sub).mkdir()
        cmd = ([sys.executable] if nproc == 1 else _torchrun(nproc, 29666)) + [me, *args, *extra]
        res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib), cwd=str(tmp_path / sub))
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    names = compare_outputs(str(tmp_path / "single" / "iisph_body_case_output"),
                            str(tmp_path / "sharded" / "iisph_body_case_output"), D)
    assert names == ["obj_2_000000.obj", "obj_2_000001.obj", "particle_object_0_000000.ply",
                     "particle_object_0_000001.ply"], names


def test_iisph_dynamic_solids_under_address_sanitizer():
    """One world-1 sharded IISPH run with the cube and the block in the ASan build of the emulated library."""
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    lib = build_emu.build(asan=True)
    out = _run(1, None, ["--counts", "12", "6", "6", "--steps", "6", "--vx", "3"], lib=lib,
               env_extra={"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"})
    assert out["same_particle_set"] and out["max_dx_over_d"] < 1e-3 and out["ok"], out
    assert out["iterations_sharded"] == out["iterations_single"], out


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["cli"])
    ap.add_argument("--scene-file", default="")
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--sharded", action="store_true")
    sys.exit(_launch_cli(ap.parse_args()) or 0)
