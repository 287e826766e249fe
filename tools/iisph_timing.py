"""IISPH and PCISPH against DFSPH on one GPU, in one run: dragon_bath_iisph, dragon_bath_dfsph and dragon_bath_pcisph
after a warm-up.

For each scene: ms/step over `--steps` device-side-loop steps (host clock around synchronised steps), pressure sweeps
per step, the last average error, and the cost of one pressure sweep alone -- `--sweeps` back-to-back sweeps timed
with CUDA events on the state of the last step (IISPH: k_iisph_pressure_accel + k_iisph_pressure_update, the error sum
fused in; DFSPH: k_dfsph_iteration<1> + k_dfsph_density_change<1>, the two list walks of a pressure sweep without the
error sum; PCISPH: k_pcisph_predict + k_pcisph_update_pressure + k_pcisph_pressure_force<false>, the error max fused
in).  The other scenes' warm-up and window are rescaled by the ratio of the time steps, so that every sweep is timed on
states at the same simulated time (the same phase of the falling block).  The card's name and
power limit are read in the same run.  Writes one JSON object to `--out` and prints it (DESIGN.md section 10 quotes
profiles/h100_iisph_timing.json, written before PCISPH existed; section 11 quotes profiles/h100_pcisph_timing.json,
written by `--steps 100 --warmup 100 --out profiles/h100_pcisph_timing.json`).

    python tools/iisph_timing.py [--steps 40] [--warmup 20] [--sweeps 50] [--out PATH]
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


def run(name, steps, warmup, sweeps, t_scale=None):
    """t_scale = (dt of the IISPH run): warm-up and timed window are rescaled to cover the same simulated time."""
    ps = ParticleSystem(SimConfig(scene.NAMED_SCENES[name]()), device="cuda:0")
    s = ps.build_solver()
    s.initialize()
    method = ps.cfg.get_cfg("simulationMethod")
    iisph, pcisph = method == 3, method == 1
    if t_scale is not None:
        f = t_scale / float(s.dt[None])
        warmup, steps = max(1, round(warmup * f)), max(1, round(steps * f))
    for _ in range(warmup):
        s.step()
    torch.cuda.synchronize()
    per_step, its, errs = [], [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        s.step()
        torch.cuda.synchronize()
        per_step.append((time.perf_counter() - t0) * 1e3)
        its.append(int(s.last_iterations))
        errs.append(float(s.last_avg_density_error if iisph else s.last_max_density_error if pcisph else 0.0))
    ps._engine.check_status()
    # one pressure sweep alone, on the state the last step left (the lists of a fresh density pass)
    ps.initialize_particle_system()
    s.compute_moving_boundary_volume()
    s.compute_densities()
    err = torch.zeros(1, dtype=torch.float64, device=ps.device)
    eng = ps._engine
    if pcisph:
        s.pci_compute_deltas()
        err_bits = torch.zeros(1, dtype=torch.int32, device=ps.device)
        delta = float(s.pci_scaling_factor())
        sweep = lambda: (eng.pcisph_op(2), eng.pcisph_op(3, delta, err_bits), eng.pcisph_op(4))  # noqa: E731
    elif iisph:
        s.compute_non_pressure_forces()
        s.predict_advection()
        sweep = lambda: eng.iisph_op(3, s.omega, err)  # noqa: E731
    else:
        s.compute_non_pressure_forces()
        s.predict_velocity()
        sweep = lambda: (eng.dfsph_op(7), eng.dfsph_op(3))  # noqa: E731
    sweep()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(sweeps):
        sweep()
    e1.record()
    torch.cuda.synchronize()
    ms_sweep = e0.elapsed_time(e1) / sweeps
    out = {"scene": name, "particles": int(ps.particle_num[None]), "dt": float(s.dt[None]), "warmup": warmup,
           "steps": steps, "simulated_window_s": [warmup * float(s.dt[None]), (warmup + steps) * float(s.dt[None])],
           "ms_per_step_mean": sum(per_step) / len(per_step), "ms_per_step": per_step,
           "pressure_sweeps_per_step": its, "ms_per_pressure_sweep": ms_sweep}
    if iisph:
        out["avg_density_error"] = errs
    elif pcisph:
        out["max_density_error"] = errs
    else:
        out["divergence_iterations_last"] = int(s.last_iterations_v)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sweeps", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_iisph_timing.json"))
    a = ap.parse_args()
    card, plimit = slab._gpu_name_and_power_limit(0)
    res = {"gpu": {"name": card, "power_limit_w": plimit}, "steps": a.steps, "warmup": a.warmup,
           "runs": [run("dragon_bath_iisph", a.steps, a.warmup, a.sweeps)]}
    res["runs"].append(run("dragon_bath_dfsph", a.steps, a.warmup, a.sweeps, t_scale=res["runs"][0]["dt"]))
    res["runs"].append(run("dragon_bath_pcisph", a.steps, a.warmup, a.sweeps, t_scale=res["runs"][0]["dt"]))
    ii, df, pc = res["runs"]
    res["sweep_ratio_iisph_over_dfsph"] = ii["ms_per_pressure_sweep"] / df["ms_per_pressure_sweep"]
    res["sweep_ratio_pcisph_over_dfsph"] = pc["ms_per_pressure_sweep"] / df["ms_per_pressure_sweep"]
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}))
    for r in res["runs"]:
        print(json.dumps({k: v for k, v in r.items() if k not in ("ms_per_step", "avg_density_error",
                                                                  "max_density_error")}))


if __name__ == "__main__":
    main()
