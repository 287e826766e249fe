"""Output of sharded runs on the CPU: ``sph_shard_dump`` / ``ShardedSimulation.dump`` and ``run_simulation.py``'s
sharded driver (``run_sharded``) in the host-emulated build of the library over gloo (``slab.GlooTransport`` stands in
for NCCL).  The gathered rows must be exactly the rows of ``gather_owned`` of the same state, in the same order, and
the sharded CLI must write the single engine's files.

This file is also the launcher of those runs: ``python tests/test_slab_gloo_dump.py MODE ...`` (under
torch.distributed.run for world > 1) with SPH_EMU_LIB pointing at the emulated library."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 0.02
SPH_E_ARG, SPH_E_CAPACITY = -1, -3


# ------------------------------------------------------------------------------------------------------------------
# the launcher (runs in the subprocesses)
# ------------------------------------------------------------------------------------------------------------------
def _install():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import emu_engine
    emu_engine.install(os.environ["SPH_EMU_LIB"])


def _dump_scene(world, dfsph):
    """The dam break (object 0) at +1.5 m/s; WCSPH: on the static floor block (object 1) with the shape-matched cube
    (object 2) on its surface."""
    from check_slab_parity import add_dynamic_solids, static_block_scene
    from sph_taichi_b200 import scene
    c = [24, 6, 6]
    if dfsph:
        sc = scene._as_dfsph(scene.dam_break_box(c, domain_end=[2.5 * c[0] * D + 0.2, c[1] * D + 0.4, c[2] * D + 0.12],
                                                 start=[0.06] * 3))
    else:
        sc = add_dynamic_solids(static_block_scene(c, D), c, D, world, True, False)
        sc["RigidBodies"][0]["translation"][1] += 0.04  # static_block_scene lifts the fluid by 0.04
    sc["FluidBlocks"][0]["velocity"] = [1.5, 0.0, 0.0]
    return sc


def _launch_dump(a):
    """Dump objects 0, 1, 2 and an absent id after a.steps steps and compare with gather_owned; capacity checks."""
    import ctypes as C

    import numpy as np
    import torch
    import torch.distributed as dist
    from sph_taichi_b200 import SimConfig, scene, slab
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    sc = _dump_scene(world, a.dfsph)
    slabs = None
    if a.skew:
        arrays = scene.assemble_particles(SimConfig(sc), 3, D)[0]
        gx = int(np.ceil(np.array(sc["Configuration"]["domainEnd"]) / (2 * D)).astype(int)[0])
        hist = np.bincount(slab.layer_of(arrays["x"], 2 * D), minlength=gx)[:gx]
        base = slab.plan_slabs(hist, world, min_width=slab.SEND_LAYERS_BODIES + 1)
        cuts = [s_[0] for s_ in base] + [base[-1][1]]
        cuts = [cuts[0]] + [c_ + a.skew for c_ in cuts[1:-1]] + [cuts[-1]]
        slabs = [(cuts[r], cuts[r + 1]) for r in range(world)]
    transport = slab.GlooTransport() if world > 1 else None
    sim, n_total = slab.build_sharded(sc, rank, world, torch.device("cpu"), rebalance_every=a.rebalance_every,
                                      slabs=slabs, transport=transport, dynamic_solids=not a.dfsph)
    first = sim.info()
    sim.step(a.steps)
    out = {"rank": rank, "objects": {}, "slab0": [first["x_lo"], first["x_hi"]]}
    last = sim.info()
    out["slab1"] = [last["x_lo"], last["x_hi"]]
    for oid in (0, 1, 2, 77):
        mine = int((sim.owned_tensors()[3] == oid).sum())
        g0 = sim.transport_stats()
        got = sim.dump(oid)
        g1 = sim.transport_stats()
        gathered = slab.gather_owned(sim)
        rec = {"mine": mine, "groups": g1[0] - g0[0], "bytes": g1[1] - g0[1],
               "bytes_formula": (world - 1) * 16 + (24 * mine if rank else 0)}
        if rank == 0:
            X, V, OID = gathered[0], gathered[1], gathered[3]
            m = OID == oid
            want = np.concatenate([X[m].numpy(), V[m].numpy()], axis=1)
            have = np.concatenate([got["position"], got["velocity"]], axis=1)
            rec.update(rows=int(have.shape[0]), count=int(sim.object_counts.get(oid, 0)),
                       same_order=bool(have.shape == want.shape and np.array_equal(have, want)))
            ks, kw = np.lexsort(have.T[::-1]), np.lexsort(want.T[::-1])
            rec["same_multiset"] = bool(have.shape == want.shape and np.array_equal(have[ks], want[kw]))
        else:
            rec["none"] = got is None
        out["objects"][str(oid)] = rec
    if a.capacity:
        # rank 0 one row short of the fluid, then (a second call) a non-root rank one row short of its own rows
        e = sim.eng
        fluid = sim.object_counts[0]
        cap = sim.n_cap if rank else fluid
        x = torch.empty((max(cap, fluid) + 1, 3), dtype=torch.float32)
        v = torch.empty_like(x)
        rows, st = C.c_int64(0), C.c_uint32(0)
        calls = []
        for short in ([0] + ([world - 1] if world > 1 else [])):
            mine = int((sim.owned_tensors()[3] == 0).sum())
            want_cap = (fluid if rank == 0 else max(mine - 1, 0)) if rank == short else (fluid if rank == 0 else sim.n_cap)
            want_cap -= 1 if rank == short == 0 else 0
            rc = e.lib.sph_shard_dump(e.ctx, 0, C.c_void_p(x.data_ptr()), C.c_void_p(v.data_ptr()), want_cap,
                                      C.byref(rows), C.byref(st), None)
            calls.append({"short": short, "rc": rc, "msg": e.lib.sph_last_error(e.ctx).decode()})
        sim.step(1)
        got = sim.dump(0)
        out["capacity"] = {"calls": calls, "after_rows": None if got is None else int(got["position"].shape[0]),
                           "fluid": fluid}
    outs = [None] * world
    if world > 1:
        dist.all_gather_object(outs, out)
        dist.destroy_process_group()
    else:
        outs = [out]
    if rank == 0:
        print(json.dumps({"ranks": outs, "n_total": int(n_total)}))


def _export_scene(kind, world):
    """The CLI scenes: "wcsph" -- the dam break (16 x 8 x 8) at rest with the shape-matched cube on its surface across
    the initial cut, exportPly + exportObj; "dfsph" -- the fluid alone, DFSPH, exportPly; "dfsph_body" -- DFSPH with
    the cube (refused)."""
    from check_slab_parity import add_dynamic_solids
    from sph_taichi_b200 import scene
    c = [16, 8, 8] if kind == "wcsph" else [24, 6, 6]
    sc = scene.dam_break_box(c, domain_end=[2.5 * c[0] * D + 0.2, c[1] * D + 0.4, c[2] * D + 0.12], start=[0.06] * 3)
    if kind in ("wcsph", "dfsph_body"):
        sc = add_dynamic_solids(sc, c, D, world, True, False)
    if kind.startswith("dfsph"):
        sc = scene._as_dfsph(sc)
    sc["Configuration"].update(exportPly=True, exportObj=kind == "wcsph")
    return sc


def _launch_cli(a):
    """run_simulation.py's loop on the scene file a.scene_file in the current directory: run_single, or run_sharded on
    WORLD_SIZE ranks over gloo.  Prints the cut and the cube's layers (the cube must straddle the cut)."""
    import numpy as np
    import torch
    import torch.distributed as dist
    from run_simulation import run_sharded, run_single
    from sph_taichi_b200 import SimConfig, scene, slab
    cfg = SimConfig(a.scene_file)
    name = os.path.basename(a.scene_file).split(".")[0]
    if not a.sharded:
        return run_single(cfg, name, a.frames, quiet=True)
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    if rank == 0:
        arrays = scene.assemble_particles(SimConfig(a.scene_file), 3, D)[0]
        gx = int(np.ceil(np.array(cfg.get_cfg("domainEnd")) / (2 * D)).astype(int)[0])
        lay = slab.layer_of(arrays["x"], 2 * D)
        dynamic = bool(cfg.get_rigid_bodies())
        width = (slab.SEND_LAYERS_BODIES if dynamic else slab.SEND_LAYERS) + 1
        slabs = slab.plan_slabs(np.bincount(lay, minlength=gx)[:gx], world, min_width=width)
        body = lay[arrays["object_id"] == 2]
        print(json.dumps({"cuts": [s_[1] for s_ in slabs[:-1]],
                          "body_layers": [int(body.min()), int(body.max()) + 1] if body.size else None}))
    try:
        return run_sharded(cfg, name, a.frames, torch.device("cpu"), transport=slab.GlooTransport() if world > 1 else None,
                           quiet=True)
    finally:
        if world > 1:
            dist.destroy_process_group()


def _launch_main(a):
    """run_simulation.py itself (its __main__), with the given arguments."""
    import runpy
    sys.argv = [os.path.join(ROOT, "run_simulation.py")] + [t for t in a.args if t != "--"]
    runpy.run_path(sys.argv[0], run_name="__main__")


def _launch_refusal(_a):
    """sph_shard_dump on a context that was never sharded, and bad arguments on a sharded one."""
    import ctypes as C

    import numpy as np
    import torch
    from sph_taichi_b200 import SimConfig, engine, scene, slab
    sc = scene.dam_break_box([8, 6, 6], domain_end=[0.6, 0.4, 0.4], start=[0.06] * 3)
    cfg = SimConfig(sc)
    arrays, _, _, counts = scene.assemble_particles(cfg, 3, D)
    n = counts["total"]
    e = engine.Engine(slab.scene_params(cfg), n_max=4 * n, n_solid=0, n_bodies=0, device=torch.device("cpu"))
    e.pack(slab.field_tensors(arrays, n, float(np.float32(0.8 * D ** 3)), torch.device("cpu")), n, 0, False)
    x = torch.zeros((n, 3), dtype=torch.float32)
    rows, st = C.c_int64(0), C.c_uint32(0)
    xp = C.c_void_p(x.data_ptr())
    rc = e.lib.sph_shard_dump(e.ctx, 0, xp, xp, n, C.byref(rows), C.byref(st), None)
    res = {"plain": [rc, e.lib.sph_last_error(e.ctx).decode()]}
    e.close()
    sim, _ = slab.build_sharded(sc, 0, 1, torch.device("cpu"))
    e = sim.eng
    res["negative_capacity"] = e.lib.sph_shard_dump(e.ctx, 0, xp, xp, -1, C.byref(rows), C.byref(st), None)
    res["null_x"] = e.lib.sph_shard_dump(e.ctx, 0, None, xp, n, C.byref(rows), C.byref(st), None)
    res["null_rows"] = e.lib.sph_shard_dump(e.ctx, 0, xp, xp, n, None, C.byref(st), None)
    res["ok"] = e.lib.sph_shard_dump(e.ctx, 0, xp, xp, n, C.byref(rows), C.byref(st), None)
    res["rows"] = int(rows.value)
    print(json.dumps(res))


def _launcher():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["dump", "cli", "main", "refusal"])
    ap.add_argument("--dfsph", action="store_true")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--skew", type=int, default=0)
    ap.add_argument("--rebalance-every", type=int, default=8)
    ap.add_argument("--capacity", action="store_true")
    ap.add_argument("--scene-file", default="")
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--sharded", action="store_true")
    a, a.args = ap.parse_known_args()  # mode "main": the arguments of run_simulation.py, after "--"
    _install()
    sys.exit({"dump": _launch_dump, "cli": _launch_cli, "main": _launch_main, "refusal": _launch_refusal}[a.mode](a) or 0)


# ------------------------------------------------------------------------------------------------------------------
# the tests
# ------------------------------------------------------------------------------------------------------------------
def _env(lib, extra=None):
    env = dict(os.environ, SPH_EMU_LIB=lib, PYTHONPATH=ROOT, SPH_SHARD_GRAPH="0", SPH_SHARD_SPLIT_DENSITY="0")
    env.pop("SPH_B200_LIB", None)
    env.update(extra or {})
    return env


def _run(nproc, port, args, lib=None, env_extra=None, cwd=ROOT, check=True):
    import build_emu
    lib = lib or build_emu.build()
    me = os.path.abspath(__file__)
    if nproc == 1:
        cmd = [sys.executable, me, *args]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
               "127.0.0.1", "--master-port", str(port), me, *args]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=_env(lib, env_extra), cwd=cwd)
    if check:
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return res


def _json(res):
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert lines, res.stdout[-2000:] + res.stderr[-2000:]
    return json.loads(lines[-1])


def _check_dump(out, world, objects=("0", "1", "2", "77")):
    ranks = out["ranks"]
    assert len(ranks) == world
    r0 = ranks[0]["objects"]
    for oid in objects:
        rec = r0[oid]
        assert rec["same_multiset"] and rec["same_order"], (oid, rec)
        assert rec["rows"] == rec["count"] == sum(r["objects"][oid]["mine"] for r in ranks), (oid, rec)
        for r in ranks:
            o = r["objects"][oid]
            assert o["bytes"] == o["bytes_formula"], (oid, r["rank"], o)
            others = any(q["objects"][oid]["mine"] for q in ranks[1:])
            assert o["groups"] == (0 if world == 1 else 1 + int(others)), (oid, r["rank"], o)
            if r["rank"]:
                assert o["none"], o
    assert r0["77"]["rows"] == 0 and r0["0"]["rows"] > 0


@pytest.fixture(autouse=True)
def _emu_path():
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    yield
    sys.path.remove(os.path.join(ROOT, "tests", "emu"))


def test_dump_two_ranks():
    """WCSPH with the static block and the cube, 2 ranks: the fluid's and the block's rows are split over both ranks."""
    out = _json(_run(2, 29641, ["dump", "--steps", "6"]))
    _check_dump(out, 2)
    ranks = out["ranks"]
    for oid in ("0", "1"):
        assert all(r["objects"][oid]["mine"] > 0 for r in ranks), (oid, ranks)


def test_dump_three_ranks_skewed_cuts_rebalanced():
    """3 ranks, every interior cut shifted by two layers and re-balanced every 2 steps."""
    out = _json(_run(3, 29642, ["dump", "--steps", "6", "--skew", "-2", "--rebalance-every", "2"]))
    _check_dump(out, 3)
    assert all(r["objects"]["0"]["mine"] > 0 for r in out["ranks"]), out["ranks"]


def test_dump_dfsph_two_ranks():
    """Sharded DFSPH, fluid only, 2 ranks (objects 1 and 2 are absent)."""
    out = _json(_run(2, 29643, ["dump", "--dfsph", "--steps", "3"]))
    _check_dump(out, 2)
    assert out["ranks"][0]["objects"]["1"]["rows"] == 0


def test_dump_capacity_refused_on_every_rank():
    """Rank 0 one row short of the fluid, then rank 1 one row short of its own rows: every rank returns
    SPH_E_CAPACITY with a message naming the capacity and none hangs; the next step and a dump then succeed."""
    out = _json(_run(2, 29644, ["dump", "--steps", "2", "--capacity"]))
    for r in out["ranks"]:
        calls = r["capacity"]["calls"]
        assert [c["short"] for c in calls] == [0, 1], calls
        for c in calls:
            assert c["rc"] == SPH_E_CAPACITY and "capacity" in c["msg"], (r["rank"], c)
        assert "rank 0 gathers" in calls[0]["msg"] and "rank 1 holds" in calls[1]["msg"], calls
    cap0 = out["ranks"][0]["capacity"]
    assert cap0["after_rows"] == cap0["fluid"] > 0, cap0


def test_dump_refused_without_sharding():
    """A context that was never sharded is refused (single-GPU contexts have sph_unpack_xv); a negative capacity
    and null pointers are argument errors."""
    out = _json(_run(1, None, ["refusal"]))
    assert out["plain"][0] == SPH_E_ARG and "sph_shard_configure was not called" in out["plain"][1], out
    assert out["negative_capacity"] == out["null_x"] == out["null_rows"] == SPH_E_ARG, out
    assert out["ok"] == 0 and out["rows"] > 0, out


def test_dump_under_address_sanitizer():
    """One world-1 dump run in the ASan build of the emulated library."""
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    lib = build_emu.build(asan=True)
    out = _json(_run(1, None, ["dump", "--steps", "2"], lib=lib,
                     env_extra={"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"}))
    _check_dump(out, 1)


def _read_ply(path):
    import numpy as np
    lines = open(path).read().splitlines()
    end = lines.index("end_header")
    n = int([ln for ln in lines[:end] if ln.startswith("element vertex")][0].split()[-1])
    pts = np.array([[float(t) for t in ln.split()] for ln in lines[end + 1:]], dtype=np.float64).reshape(-1, 3)
    assert pts.shape == (n, 3)
    return pts


def _read_obj(path):
    import numpy as np
    lines = open(path).read().splitlines()
    return np.array([[float(t) for t in ln.split()[1:]] for ln in lines if ln.startswith("v ")]), \
        [ln for ln in lines if ln.startswith("f ")]


def compare_outputs(single_dir, sharded_dir, d):
    """The output files of two runs of one scene: identical names, every PLY frame a nearest-neighbour bijection within
    1e-3 d, OBJ vertices within 1e-3 d and identical faces.  Returns the file names."""
    import numpy as np
    from scipy.spatial import cKDTree
    names = sorted(os.listdir(single_dir))
    assert names == sorted(os.listdir(sharded_dir)), (names, sorted(os.listdir(sharded_dir)))
    for n in names:
        if n.endswith(".ply"):
            a, b = _read_ply(os.path.join(single_dir, n)), _read_ply(os.path.join(sharded_dir, n))
            assert a.shape == b.shape and a.shape[0] > 0, (n, a.shape, b.shape)
            dist_, idx = cKDTree(a).query(b, k=1)
            assert dist_.max() <= 1e-3 * d, (n, dist_.max() / d)
            assert np.array_equal(np.sort(idx), np.arange(a.shape[0])), n  # one-to-one
        elif n.endswith(".obj"):
            (va, fa), (vb, fb) = _read_obj(os.path.join(single_dir, n)), _read_obj(os.path.join(sharded_dir, n))
            assert fa == fb and va.shape == vb.shape and va.size, n
            assert np.abs(va - vb).max() <= 1e-3 * d, (n, np.abs(va - vb).max() / d)
    return names


def _cli_pair(tmp_path, kind, world, frames, port):
    sc_dir = tmp_path / "scene"
    sc_dir.mkdir()
    import_code = (f"import sys, json; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tools')!r}]; "
                   f"from tests.test_slab_gloo_dump import _export_scene; "
                   f"json.dump(_export_scene({kind!r}, {world}), open({str(sc_dir / 'export_case.json')!r}, 'w'))")
    subprocess.run([sys.executable, "-c", import_code], check=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT)
    scene_file = str(sc_dir / "export_case.json")
    single, sharded = tmp_path / "single", tmp_path / "sharded"
    single.mkdir(); sharded.mkdir()
    _run(1, None, ["cli", "--scene-file", scene_file, "--frames", str(frames)], cwd=str(single))
    res = _run(world, port, ["cli", "--sharded", "--scene-file", scene_file, "--frames", str(frames)], cwd=str(sharded))
    return (compare_outputs(str(single / "export_case_output"), str(sharded / "export_case_output"), D),
            json.loads([ln for ln in res.stdout.splitlines() if ln.startswith("{")][0]))


def test_cli_two_ranks_wcsph_ply_and_obj(tmp_path):
    """run_sharded on 2 ranks against run_single, WCSPH with the cube across the cut: 41 steps, exports after
    render updates 0 and 40 (output_interval = int(0.016 / 4e-4))."""
    names, meta = _cli_pair(tmp_path, "wcsph", 2, 41, 29645)
    assert names == ["obj_2_000000.obj", "obj_2_000001.obj", "particle_object_0_000000.ply",
                     "particle_object_0_000001.ply"], names
    lo, hi = meta["body_layers"]
    assert lo < meta["cuts"][0] < hi, meta


def test_cli_three_ranks_dfsph_ply(tmp_path):
    """run_sharded on 3 ranks against run_single, DFSPH fluid only: 9 steps, exports after render updates 0, 4, 8
    (output_interval = int(0.016 / 4e-3))."""
    names, _meta = _cli_pair(tmp_path, "dfsph", 3, 9, 29646)
    assert names == [f"particle_object_0_{k:06}.ply" for k in range(3)], names


def test_cli_refuses_dfsph_with_dynamic_body(tmp_path):
    """run_simulation.py --gpus 1 on a DFSPH scene with a shape-matched body exits non-zero with the message."""
    code = (f"import sys, json; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tools')!r}]; "
            f"from tests.test_slab_gloo_dump import _export_scene; "
            f"json.dump(_export_scene('dfsph_body', 1), open({str(tmp_path / 'dfsph_body.json')!r}, 'w'))")
    subprocess.run([sys.executable, "-c", code], check=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT)
    res = _run(1, None, ["main", "--", "--scene_file", str(tmp_path / "dfsph_body.json"), "--gpus", "1", "--frames", "1"],
               cwd=str(tmp_path), check=False)
    assert res.returncode != 0 and "WCSPH only" in res.stderr, res.stdout[-2000:] + res.stderr[-2000:]


if __name__ == "__main__":
    _launcher()
