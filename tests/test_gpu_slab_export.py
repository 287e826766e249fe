"""Output of sharded runs on the GPU: ``ShardedSimulation.dump`` of the full-size dragon_bath against the plain
engine's ``ParticleSystem.dump``, and ``run_simulation.py --gpus N`` against the single-GPU ``run_simulation.py`` on
the export scene of tests/test_exporters.py (fluid with a falling shape-matched cube, exportPly + exportObj)."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_dragon_bath_single_rank_dump_equals_plain_engine():
    """World 1, the whole dragon_bath for 40 WCSPH steps: object 0's rows of sim.dump(0) are ps.dump(0)'s rows, as
    exact row multisets; the JSON line also says whether the row order is the same."""
    code = textwrap.dedent("""
        import json, numpy as np, torch
        from sph_taichi_b200 import ParticleSystem, SimConfig, scene, slab
        dev = torch.device("cuda:0")
        sc = scene.dragon_bath()
        sim, _ = slab.build_sharded(sc, 0, 1, dev)
        sim.step(40)
        got = sim.dump(0)
        del sim
        ps = ParticleSystem(SimConfig(sc), device=dev)
        solver = ps.build_solver()
        solver.initialize()
        solver.step(40)
        want = ps.dump(0)
        a = np.concatenate([got["position"], got["velocity"]], axis=1)
        b = np.concatenate([want["position"], want["velocity"]], axis=1)
        same_shape = a.shape == b.shape
        ka, kb = np.lexsort(a.T[::-1]), np.lexsort(b.T[::-1])
        print(json.dumps({"rows": a.shape[0], "rows_plain": b.shape[0],
                          "same_multiset": bool(same_shape and np.array_equal(a[ka], b[kb])),
                          "same_order": bool(same_shape and np.array_equal(a, b))}))
    """)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1500,
                         env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    out = json.loads(lines[-1])
    print(out)
    assert out["rows"] == out["rows_plain"] > 400000, out
    assert out["same_multiset"], out


def _export_scene_file(tmp_path):
    from tests.test_exporters import _export_scene
    f = tmp_path / "export_case.json"
    f.write_text(json.dumps(_export_scene()))
    return str(f)


def _cli(cwd, scene_file, frames, nproc=None, port=29661):
    args = [os.path.join(ROOT, "run_simulation.py"), "--scene_file", scene_file, "--frames", str(frames), "--quiet"]
    if nproc is None:
        cmd = [sys.executable, *args]
    elif nproc == 1:
        cmd = [sys.executable, *args, "--gpus", "1"]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), *args, "--gpus", str(nproc)]
    os.makedirs(cwd, exist_ok=True)
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=cwd, env=dict(os.environ, PYTHONPATH=ROOT))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    return os.path.join(cwd, "export_case_output")


def _cli_against_single(tmp_path, nproc):
    from tests.test_slab_gloo_dump import compare_outputs
    scene_file = _export_scene_file(tmp_path)
    frames = 81  # output_interval = int(0.016 / 4e-4) = 40 render updates -> exports at update 0, 40, 80
    single = _cli(str(tmp_path / "single"), scene_file, frames)
    sharded = _cli(str(tmp_path / "sharded"), scene_file, frames, nproc=nproc)
    names = compare_outputs(single, sharded, 0.02)
    assert names == [f"obj_1_{k:06}.obj" for k in range(3)] + [f"particle_object_0_{k:06}.ply" for k in range(3)], names


def test_cli_one_gpu_sharded_equals_single(tmp_path):
    _cli_against_single(tmp_path, 1)


def test_cli_two_gpus_sharded_equals_single(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _cli_against_single(tmp_path, 2)
