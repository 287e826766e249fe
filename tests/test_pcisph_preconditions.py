"""The refusal contract of the PCISPH entry points on the host-emulated build, and of the existing entry points on a
PCISPH context: the PCISPH calls refuse a context of another solver (an IISPH one with the IISPH context's message)
and a sharded one; the WCSPH, DFSPH and IISPH
calls and every sph_shard_configure* call refuse a PCISPH context (PCISPH is single-GPU); sph_set_pcisph(1) is
refused on a sharded context and sph_set_pcisph(0) leaves a context of another solver as it is.

This file is also the launcher of the checks: ``python tests/test_pcisph_preconditions.py run`` with SPH_EMU_LIB
pointing at the emulated library."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))

OK, E_ARG = 0, -1
PCISPH_CONTEXT = "this context is in PCISPH mode (sph_set_pcisph): it steps with sph_pcisph_op"
SINGLE_GPU = "PCISPH (sph_set_pcisph) is single-GPU: x-slab sharding runs WCSPH, DFSPH and IISPH contexts"
NO_PCISPH = "sph_set_pcisph(1) was not called"
NOT_CONFIGURED = "sph_shard_configure was not called"
IISPH_CONTEXT = "this context is in IISPH mode (sph_set_iisph): it steps with sph_iisph_op"
STALE = "neighbour structure is stale: call sph_neighbor_build first"
STALE_LISTS = "neighbour lists are stale: run sph_neighbor_build and op 0"

STATES = ("wcsph", "dfsph", "iisph", "pcisph", "static_wcsph")
PCISPH_CALLS = ("sph_pcisph_op", "sph_pcisph_solve", "sph_pcisph_step", "sph_pcisph_read")


def expect(state, entry):
    """(return code, message) of `entry` on a context in `state`; message None: a bare code."""
    pc = state == "pcisph"
    if entry in PCISPH_CALLS:
        if not pc:
            return E_ARG, IISPH_CONTEXT if state == "iisph" else NO_PCISPH
        return {"sph_pcisph_op": (E_ARG, STALE), "sph_pcisph_solve": (E_ARG, STALE_LISTS)}.get(entry, (OK, None))
    if entry in ("sph_pcisph_step(-1)", "sph_pcisph_solve(max_iterations=0)"):
        return E_ARG, None  # the bare argument checks come before the solver's
    if entry == "sph_set_pcisph(1)":
        return (E_ARG, SINGLE_GPU) if state == "static_wcsph" else (OK, None)
    if entry == "sph_set_pcisph(0)":
        return OK, None
    if not pc:
        return None  # the existing calls on the other states: tests/test_entry_preconditions.py
    if entry in ("sph_step", "sph_dfsph_op", "sph_dfsph_solve", "sph_dfsph_step", "sph_iisph_op", "sph_iisph_solve",
                 "sph_iisph_step", "sph_iisph_read"):
        return E_ARG, PCISPH_CONTEXT
    if entry in ("sph_shard_configure", "sph_shard_configure_bodies", "sph_shard_configure_iisph_bodies"):
        return E_ARG, SINGLE_GPU
    if entry in ("sph_shard_step", "sph_shard_dfsph_step", "sph_shard_iisph_step", "sph_shard_begin"):
        return E_ARG, NOT_CONFIGURED
    raise KeyError(entry)


ENTRIES = list(PCISPH_CALLS) + [
    "sph_pcisph_step(-1)", "sph_pcisph_solve(max_iterations=0)", "sph_set_pcisph(1)", "sph_set_pcisph(0)",
    "sph_step", "sph_dfsph_op", "sph_dfsph_solve", "sph_dfsph_step", "sph_iisph_op", "sph_iisph_solve",
    "sph_iisph_step", "sph_iisph_read", "sph_shard_configure", "sph_shard_configure_bodies",
    "sph_shard_configure_iisph_bodies", "sph_shard_step", "sph_shard_dfsph_step", "sph_shard_iisph_step",
    "sph_shard_begin",
]
MUTATING = {"sph_set_pcisph(1)", "sph_set_pcisph(0)"}


def run_checks():
    import ctypes as C

    import emu_engine
    emu_engine.install(os.environ["SPH_EMU_LIB"])
    import numpy as np
    import torch
    from sph_taichi_b200 import SimConfig, _lib, engine, scene, slab

    cpu = torch.device("cpu")
    cfg = SimConfig(scene.dam_break_box([6, 4, 4], domain_end=[0.6, 0.3, 0.3], start=[0.06] * 3))
    params = slab.scene_params(cfg)
    gx = int(params.grid_num[0])
    arrays, _, _, counts = scene.assemble_particles(cfg, 3, 0.02)
    n = counts["total"]
    m_V0 = float(np.float32(0.8 * 0.02 ** 3))

    def state(name):
        e = engine.Engine(params, n_max=4 * n, n_solid=8, n_bodies=1, device=cpu)
        e.pack(slab.field_tensors(arrays, n, m_V0, cpu), n, 0, False)
        lib, ctx = e.lib, e.ctx
        if name == "dfsph":
            assert lib.sph_set_dfsph(ctx, 1) == OK
        if name == "iisph":
            assert lib.sph_set_iisph(ctx, 1) == OK
        if name == "pcisph":
            assert lib.sph_set_pcisph(ctx, 1) == OK
        if name == "static_wcsph":
            assert lib.sph_shard_configure(ctx, 0, gx, 1, n, 0) == OK, lib.sph_last_error(ctx)
        return e

    dio = _lib.SphDfsphStep(n_fluid=1, max_iterations=1, max_iterations_v=1, first_batch=1, first_batch_v=1)
    iio = _lib.SphIisphStep(max_iterations=1, omega=0.5, eta=1e-3, n_fluid=1, first_batch=1)
    pio = _lib.SphPcisphStep(delta=1.0, eta=0.01, min_iterations=3, max_iterations=1, first_batch=1)
    calls = {
        "sph_pcisph_op": lambda L, c: L.sph_pcisph_op(c, 1, 0.0, None, None),
        "sph_pcisph_solve": lambda L, c: L.sph_pcisph_solve(c, 1.0, 0.01, 3, 1, 1, None, None, None),
        "sph_pcisph_step": lambda L, c: L.sph_pcisph_step(c, 0, C.byref(pio), None),
        "sph_pcisph_read": lambda L, c: L.sph_pcisph_read(c, None, None, None, None),
        "sph_pcisph_step(-1)": lambda L, c: L.sph_pcisph_step(c, -1, C.byref(pio), None),
        "sph_pcisph_solve(max_iterations=0)": lambda L, c: L.sph_pcisph_solve(c, 1.0, 0.01, 3, 0, 1, None, None, None),
        "sph_set_pcisph(1)": lambda L, c: L.sph_set_pcisph(c, 1),
        "sph_set_pcisph(0)": lambda L, c: L.sph_set_pcisph(c, 0),
        "sph_step": lambda L, c: L.sph_step(c, 0, None),
        "sph_dfsph_op": lambda L, c: L.sph_dfsph_op(c, 0, 0.0, None, None),
        "sph_dfsph_solve": lambda L, c: L.sph_dfsph_solve(c, 1, 1, 1e-3, 0.0, 1, 1, None, None, None, None),
        "sph_dfsph_step": lambda L, c: L.sph_dfsph_step(c, 0, C.byref(dio), None),
        "sph_iisph_op": lambda L, c: L.sph_iisph_op(c, 0, 0.0, None, None),
        "sph_iisph_solve": lambda L, c: L.sph_iisph_solve(c, 1, 0.5, 1e-3, 1, 1, None, None, None),
        "sph_iisph_step": lambda L, c: L.sph_iisph_step(c, 0, C.byref(iio), None),
        "sph_iisph_read": lambda L, c: L.sph_iisph_read(c, None, None, None, None),
        "sph_shard_configure": lambda L, c: L.sph_shard_configure(c, 0, gx, 1, n, 0),
        "sph_shard_configure_bodies": lambda L, c: L.sph_shard_configure_bodies(c, 0, gx, 3, n, 0, None, 0),
        "sph_shard_configure_iisph_bodies": lambda L, c: L.sph_shard_configure_iisph_bodies(c, 0, gx, 3, n, 0, None,
                                                                                            0),
        "sph_shard_step": lambda L, c: L.sph_shard_step(c, 0, None),
        "sph_shard_dfsph_step": lambda L, c: L.sph_shard_dfsph_step(c, 0, C.byref(dio), None),
        "sph_shard_iisph_step": lambda L, c: L.sph_shard_iisph_step(c, 0, C.byref(iio), None),
        "sph_shard_begin": lambda L, c: L.sph_shard_begin(c, None),
    }
    assert set(calls) == set(ENTRIES)
    bad, cells = [], 0
    for name in STATES:
        shared = state(name)
        for entry in ENTRIES:
            want = expect(name, entry)
            if want is None:
                continue
            e = state(name) if want[0] == OK and entry in MUTATING else shared
            before = e.lib.sph_last_error(e.ctx).decode()
            rc = calls[entry](e.lib, e.ctx)
            msg = e.lib.sph_last_error(e.ctx).decode()
            code, text = want
            ok = rc == code and (msg == before if text is None and rc != OK else text is None or text in msg)
            cells += 1
            if not ok:
                bad.append(f"{name} / {entry}: got {(rc, msg)}, want {want}")
            if e is not shared:
                e.close()
        shared.close()
    # the transitions: sph_set_pcisph(0) leaves another solver's context alone, and leaves PCISPH for WCSPH
    for name, after in (("dfsph", "sph_dfsph_op"), ("iisph", "sph_iisph_read"), ("pcisph", "sph_step")):
        e = state(name)
        lib, ctx = e.lib, e.ctx
        assert lib.sph_set_pcisph(ctx, 0) == OK
        rc = calls[after](lib, ctx)
        msg = lib.sph_last_error(ctx).decode()
        cells += 1
        if (name == "dfsph" and (rc, msg[:len(STALE)]) != (E_ARG, STALE)) or (name != "dfsph" and rc != OK):
            bad.append(f"sph_set_pcisph(0) on {name}, then {after}: got {(rc, msg)}")
        e.close()
    # a PCISPH context keeps refusing the configure after a refusal, and sph_set_iisph(1) leaves PCISPH for IISPH
    e = state("pcisph")
    lib, ctx = e.lib, e.ctx
    assert lib.sph_set_iisph(ctx, 1) == OK and lib.sph_iisph_read(ctx, None, None, None, None) == OK
    cells += 1
    if lib.sph_pcisph_read(ctx, None, None, None, None) != E_ARG or IISPH_CONTEXT not in lib.sph_last_error(ctx).decode():
        bad.append("sph_set_iisph(1) did not leave PCISPH mode")
    e.close()
    for line in bad:
        print(line)
    print(f"{cells} cells, {len(bad)} wrong")
    return 1 if bad else 0


def test_pcisph_refusal_contract():
    import build_emu
    env = dict(os.environ, SPH_EMU_LIB=build_emu.build(), PYTHONPATH=ROOT)
    env.pop("SPH_B200_LIB", None)
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "run"], capture_output=True, text=True,
                         timeout=1500, env=env, cwd=ROOT)
    tail = res.stdout[-6000:] + res.stderr[-3000:]
    assert res.returncode == 0 and ", 0 wrong" in res.stdout, tail
    cells = int(res.stdout.split(" cells,")[0].split()[-1])
    assert cells > 50, tail


if __name__ == "__main__":
    if sys.argv[1:] != ["run"]:
        sys.exit("usage: test_pcisph_preconditions.py run")
    sys.exit(run_checks())
