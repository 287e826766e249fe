"""Sharded IISPH (or PCISPH, `--pcisph`) at world 1 against the plain engine of the same solver, on one GPU, in one
process.

Both engines run `--scene` (default dragon_bath_iisph) from the same start.  After `--warmup` steps each, the timed
window is `--rounds` rounds of `--steps` steps, alternating plain and sharded, so that both are timed on states at the
same simulated times and under the same clocks.  Per round and engine: ms/step (host clock around synchronised
steps, one step per call) and the pressure sweeps of every step.  The sharded step adds the ghost alignment, one read
of the live count and the rank-ordered loop check to the plain one; at world 1 it has no neighbours, so it sends
nothing.  The card's name and power limit are read in the same run.  Writes one JSON object to `--out` (default
profiles/h100_shard_iisph_timing.json) and prints a summary line.

`--bodies` times sharded IISPH with dynamic solids instead (scene armadillo_bath_dynamic_iisph, built with
`build_sharded(iisph_bodies=True)`; default output profiles/h100_shard_iisph_bodies_timing.json): the sharded step then
also rebuilds the solid-id slot map, computes the moving boundary volumes through it, gathers the reactions instead of
scattering them and solves the bodies from the packed table of their particles.

`--pcisph` times sharded PCISPH instead (scene dragon_bath_pcisph, built with `build_sharded(pcisph=True)`; default
output profiles/h100_shard_pcisph_timing.json): the sweeps are prediction-correction sweeps, and the sharded loop
check takes the max of the ranks' error partials.

    python tools/shard_iisph_timing.py [--bodies | --pcisph] [--steps 20] [--rounds 5] [--warmup 30] [--out PATH]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from sph_taichi_b200 import ParticleSystem, SimConfig, scene, slab  # noqa: E402


def timed(step, last_sweeps, k):
    """k steps, one per call; returns (ms per step, sweeps of every step)."""
    ms, sweeps = [], []
    for _ in range(k):
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
        sweeps.append(last_sweeps())
    return ms, sweeps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default=None, help="default: dragon_bath_iisph, with --bodies "
                                                  "armadillo_bath_dynamic_iisph, with --pcisph dragon_bath_pcisph")
    mode = ap.add_mutually_exclusive_group()
    mode.add_argument("--bodies", action="store_true", help="a scene with dynamic solids: build_sharded(iisph_bodies=True)")
    mode.add_argument("--pcisph", action="store_true", help="a PCISPH scene: build_sharded(pcisph=True)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    kind = "pcisph" if a.pcisph else "iisph_bodies" if a.bodies else "iisph"
    a.scene = a.scene or {"pcisph": "dragon_bath_pcisph", "iisph_bodies": "armadillo_bath_dynamic_iisph",
                          "iisph": "dragon_bath_iisph"}[kind]
    a.out = a.out or os.path.join(ROOT, "profiles", f"h100_shard_{kind}_timing.json")
    dev = torch.device("cuda:0")
    sc = scene.NAMED_SCENES[a.scene]()
    ps = ParticleSystem(SimConfig(sc), device=dev)
    solver = ps.build_solver()
    solver.initialize()
    opt_in = {"pcisph": True} if a.pcisph else {"iisph": True, "iisph_bodies": a.bodies}
    sim, n_total = slab.build_sharded(scene.NAMED_SCENES[a.scene](), 0, 1, dev, **opt_in)
    engines = {"plain": (lambda: solver.step(1), lambda: int(solver.last_iterations)),
               "sharded_world1": (lambda: sim.step(1), lambda: int(sim.last_iterations))}
    for step, _ in engines.values():
        for _ in range(a.warmup):
            step()
    torch.cuda.synchronize()
    rounds = {k: [] for k in engines}
    for _ in range(a.rounds):
        for name, (step, sweeps) in engines.items():
            ms, sw = timed(step, sweeps, a.steps)
            rounds[name].append({"ms_per_step": sum(ms) / len(ms), "sweeps_per_step": sum(sw) / len(sw),
                                 "sweeps": sw})
    ps._engine.check_status()
    sim.info()  # raises on a status flag
    card, plimit = slab._gpu_name_and_power_limit(0)
    dt = float(sc["Configuration"]["timeStepSize"])
    res = {"gpu": {"name": card, "power_limit_w": plimit, "read": "nvidia-smi, same run"}, "scene": a.scene,
           "particles": int(n_total), "dt": dt, "warmup": a.warmup, "steps_per_round": a.steps, "rounds": rounds,
           "simulated_window_s": [a.warmup * dt, (a.warmup + a.rounds * a.steps) * dt],
           "timing": "host clock around each synchronised step (one step per call); the engines alternate round by "
                     "round on the same GPU"}
    summary = {}
    for name, rs in rounds.items():
        ms = sorted(r["ms_per_step"] for r in rs)
        summary[name] = {"ms_per_step_median_round": ms[len(ms) // 2], "ms_per_step_rounds": ms,
                         "sweeps_per_step_mean": sum(r["sweeps_per_step"] for r in rs) / len(rs)}
    summary["sharded_over_plain"] = (summary["sharded_world1"]["ms_per_step_median_round"] /
                                     summary["plain"]["ms_per_step_median_round"])
    res["summary"] = summary
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(dict(summary, gpu=res["gpu"], particles=res["particles"])))


if __name__ == "__main__":
    main()
