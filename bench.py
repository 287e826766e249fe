#!/usr/bin/env python
"""bench.py -- WCSPH step throughput on H100 (DESIGN.md section 6).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--scene NAME] [--dump-outputs DIR]

One "step" is one full ``SPHBase.step()`` (neighbour build + density + forces + integration +
walls, sph_base.py:263-271 of the reference) over the named scene.  N = 1 runs BASELINE config 2
(dragon_bath, 423 500 fluid + 18 496 static rigid particles); N = 2/4 run the 4 M box and N = 8 the
16 M box, x-slab sharded (BASELINE configs 4/5).

Printed JSON (rank 0, one line): value = steps/s with the state resident in HBM and the L2
flushed between timed steps; ``steady`` = back-to-back steps (state L2-resident, the way a
simulation actually runs); ``e2e`` = the same through the public Python surface with pinned HOST
buffers (H2D of x, v and D2H of x, v every step); ``roofline`` for the force kernel;
``cpu_baseline`` = the CPU oracle port on this box's cores (bounded sample).

--dump-outputs DIR (single GPU) writes the state after the last step of the first timed window (x, v,
density, pressure and the rest position x_0, float32, rows ordered by (object_id, x_0)) as DIR/<name>.npy,
so that two builds can be compared output for output on the same seeded scene.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pin_openmp_for_the_cpu_arm():
    """The CPU arm pins its OpenMP threads (must happen before libgomp initialises, i.e. before torch or the oracle are
    imported); the thread COUNT is chosen in best_thread_count.  NEVER in a multi-rank run: with OMP_NUM_THREADS=1
    (torchrun's default) the binding pins the main thread of EVERY rank to the first place -- all ranks time-slice one
    core and the asynchronous launches of a sharded step crawl."""
    os.environ.setdefault("OMP_PROC_BIND", "close")
    os.environ.setdefault("OMP_PLACES", "cores")

METRIC = "M particle-updates/sec (SPH steps/sec x particles)"
UNIT = "M particle-updates/s"
FORCE_BYTES_PER_PARTICLE = 52  # SURVEY.md section 8d: algorithmic bytes of the force pass
HBM_FALLBACK_GBS = 3350.0      # H100 SXM data sheet (HBM3)


def scene_for(n_gpus, name=None):
    from sph_taichi_b200 import scene
    if name is None:
        name = {1: "dragon_bath", 2: "box_4m", 4: "box_4m", 8: "box_16m"}.get(n_gpus, "box_16m")
    return name, scene.NAMED_SCENES[name]()


def workload_config(name, sc, particles, fluid_particles):
    """The `config` object -- identical (keys AND values) in the GPU arm and in the --impl reference arm."""
    import numpy as np
    c = sc["Configuration"]
    ds = np.array(c["domainEnd"], dtype=np.float64) - np.array(c["domainStart"], dtype=np.float64)
    cells = int(np.prod(np.ceil(ds / (4.0 * c["particleRadius"])).astype(int)))
    return {"workload": name, "particles": int(particles), "fluid_particles": int(fluid_particles), "grid_cells": cells,
            "solver": "WCSPH" if c["simulationMethod"] == 0 else "DFSPH", "dt": c["timeStepSize"],
            "state": "the scene after `warmup` steps from its initial lattice",
            "l2": "GPU arm: L2 flushed between timed steps at N = 1 (256 MiB write; 'steady' is un-flushed), per-rank "
                  "working set > L2 at N > 1; reference arm: CPU caches not flushed",
            "parallelism": "GPU arm: N = 1 single GPU, N > 1 x-slabs with one halo exchange per step; reference arm: "
                           "OpenMP over the host cores"}


def measured_hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        with open(p) as fh:
            return float(json.load(fh)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return HBM_FALLBACK_GBS, "fallback (H100 SXM data sheet)"


def ncu_dram_traffic(workload, kernel):
    """dram__bytes_read.sum + dram__bytes_write.sum of one kernel, per launch, from a committed
    ncu --set full capture of the same workload (profiles/dram_traffic.json names the capture), else None."""
    try:
        with open(os.path.join(ROOT, "profiles", "dram_traffic.json")) as fh:
            return json.load(fh).get(workload, {}).get(kernel)
    except Exception:
        return None


# algorithmic bytes per particle and launch (SURVEY.md section 8d) and the compute-side model of the pair kernels:
# fp32 lane-operations = candidate tests x 7 (3 FADD + 3 FFMA + 1 SHF) + accepted pairs x the SASS instructions of
# one pair (density hit 30, force pair 54), against SMs x 128 fp32 lanes x the SM clock seen during the run
ALGO_BYTES = {"density": 24, "force": FORCE_BYTES_PER_PARTICLE}
LANE_OPS_PER_TEST, LANE_OPS_PER_DENSITY_HIT, LANE_OPS_PER_FORCE_PAIR = 7, 30, 54
KERNEL_NAME = {"density": "density pass (k_density_*: scan + neighbour lists + EOS)",
               "force": "k_force_packed<4,128,true> (cohesion + viscosity + pressure gradient + integration + walls)"}


def roofline_entry(kind, workload, n, launch_ms, total_ms, peak, work, sm_mhz, sms):
    ach = ALGO_BYTES[kind] * n / (launch_ms * 1e-3) / 1e9 if launch_ms > 0 else 0.0
    e = {"kernel": KERNEL_NAME[kind], "bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s",
         "frac": ach / peak, "traffic": ncu_dram_traffic(workload, kind),
         "algorithmic_bytes_per_particle": ALGO_BYTES[kind], "avg_launch_ms": launch_ms,
         "share_of_step": launch_ms / max(total_ms, 1e-9)}
    if work and "candidate_tests_per_pass" in work and sm_mhz:
        ops = (work["candidate_tests_per_pass"] * LANE_OPS_PER_TEST + work["accepted_pairs_per_pass"] * LANE_OPS_PER_DENSITY_HIT
               if kind == "density" else work["accepted_pairs_per_pass"] * LANE_OPS_PER_FORCE_PAIR)
        lane_peak = sms * 128 * sm_mhz * 1e6
        e["compute_side"] = {"fp32_lane_ops_per_launch": int(ops), "achieved_lane_ops_per_s": ops / (launch_ms * 1e-3),
                             "peak_lane_ops_per_s": lane_peak, "frac": ops / (launch_ms * 1e-3) / lane_peak,
                             "formula": f"density: tests x 7 + pairs x 30; force: pairs x 54; peak = {sms} SMs x 128 lanes x SM clock"}
    return e



class ClockSampler:
    """SM clock and throttle reasons sampled WHILE the timed region runs.

    In-process NVML (pynvml) from a thread, one cheap query pair every 10 ms: `nvidia-smi -lms 20` as a child process
    stalled the sampled GPU for milliseconds per poll -- invisible in a long region, but large on the short timed
    region of a sharded run.  Falls back to `nvidia-smi -lms 100` without pynvml."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")
    BITS = {"hw_slowdown": 0x8, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20, "sw_power_cap": 0x4}

    def __init__(self, index=0):
        """Construct EARLY (before the warm-up): nvmlInit enumerates the devices and stalls them -- it must
        not fall into the timed region (it would dominate a timed region of a few ms)."""
        self.rows, self.sm, self.reasons = [], [], set()
        self.proc = self.thread = self.nvml = None
        self.index = index
        self.max_mhz = None
        self._stop = threading.Event()
        try:
            import pynvml
            pynvml.nvmlInit()
            visible = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(visible.split(",")[index]) if visible and visible.split(",")[index].isdigit() else index
            h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)  # first query outside the timed region too
            self.nvml = (pynvml, h)
        except Exception:
            self.nvml = None

    def start(self):
        if self.nvml is not None:
            pynvml, h = self.nvml

            def poll():
                mode = os.environ.get("SPH_BENCH_SAMPLER", "both")  # experiments: "clock", "reasons", "both"
                period = float(os.environ.get("SPH_BENCH_SAMPLER_PERIOD_S", "0.010"))
                while not self._stop.is_set():
                    try:
                        if mode != "reasons":
                            self.sm.append(float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)))
                        if mode != "clock":
                            r = int(pynvml.nvmlDeviceGetCurrentClocksEventReasons(h))
                            for name, bit in self.BITS.items():
                                if r & bit:
                                    self.reasons.add(name)
                    except Exception:
                        pass
                    self._stop.wait(period)

            self.thread = threading.Thread(target=poll, daemon=True)
            self.thread.start()
            return
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                 "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
            time.sleep(1.0)  # nvidia-smi's start-up (NVML init, enumeration) must not fall into the timed region
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.thread is not None:
            self._stop.set()
            self.thread.join(timeout=1.0)
            sm = sorted(self.sm)
            return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": self.max_mhz, "samples": len(sm),
                    "reasons": sorted(self.reasons), "source": "NVML in-process, 10 ms period"}
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            f = [t.strip() for t in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for nm, val in zip(names, f[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(nm)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons), "source": "nvidia-smi -lms 100"}


def best_thread_count(o, reps=3):
    """Give the CPU arm its best shot: the pair loops are memory-latency bound and SMT siblings can hurt, so
    time `reps` steps (after one step) at cpu_count / 8, / 4, / 2 and cpu_count threads (plus the cgroup CPU quota when the
    box has one: a host can expose many more threads than it schedules) and keep the fastest.  Returns
    (best, {threads: steps/s}) -- timing ONE step per candidate picked different counts on equal hosts."""
    from oracle.sph_oracle import set_threads
    total = os.cpu_count() or 1
    table = {}
    cand = {total, max(1, total // 2), max(1, total // 4), max(1, total // 8)}
    quota = cgroup_cpu_quota()
    if quota:
        cand.add(max(1, min(total, int(quota))))
    # ascending, and stop at the first count whose FIRST step is already twice as slow as the best so far: past the
    # cores the box really schedules, more threads only get worse, and on the 16 M-particle scene of the 8-GPU
    # reference arm one such step costs a minute
    best_step = None
    for n in sorted(cand):
        set_threads(n)
        t0 = time.perf_counter()
        o.step()
        first = time.perf_counter() - t0
        if best_step is not None and first > 2.0 * best_step:
            table[n] = 1.0 / first
            break
        t0 = time.perf_counter()
        for _ in range(reps):
            o.step()
        per = (time.perf_counter() - t0) / reps
        table[n] = 1.0 / per
        best_step = per if best_step is None else min(best_step, per)
    best = max(table, key=table.get)
    set_threads(best)
    return best, table


def cgroup_cpu_quota():
    """CPUs the container may use per the cgroup-v2/v1 bandwidth controller (None = unlimited or unreadable)."""
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        return None if q == "max" else float(q) / float(per)
    except (OSError, ValueError):
        pass
    try:
        q = float(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
        per = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
        return None if q <= 0 else q / per
    except (OSError, ValueError):
        return None


def thread_note(best, table):
    ranked = sorted(table.items(), key=lambda kv: -kv[1])
    quota = cgroup_cpu_quota()
    return (f"OpenMP (OMP_PROC_BIND={os.environ.get('OMP_PROC_BIND')}, OMP_PLACES={os.environ.get('OMP_PLACES')}) on {best} of "
            f"{os.cpu_count()} host threads (cgroup CPU quota: {quota if quota else 'none'}); candidates timed over 3 steps each: "
            + ", ".join(f"{n} thr {v:.1f} steps/s" for n, v in ranked))


def time_cpu_oracle(scene_dict, budget_s=20.0, max_steps=200):
    """The reference's algorithm on the host cores (CPU oracle port; fp32, OpenMP)."""
    from oracle.sph_oracle import OracleSim
    o = OracleSim(scene_dict)
    o.initialize()
    cores, table = best_thread_count(o)
    t0 = time.perf_counter()
    o.step()
    t1 = time.perf_counter() - t0
    k = int(max(2, min(max_steps, budget_s / max(t1, 1e-6))))
    t0 = time.perf_counter()
    for _ in range(k):
        o.step()
    dt = time.perf_counter() - t0
    return {"value": k / dt * o.n / 1e6, "unit": UNIT, "steps_per_s": k / dt, "cores": cores, "kind": "port",
            "threads_tried": {str(n): round(v, 2) for n, v in table.items()},
            "sample": f"{k} full steps of the same scene ({o.n} particles) after the thread-count probe; "
                      + thread_note(cores, table) + "; restatement of the reference kernels, not Taichi's ti.cpu codegen"}, o.n


def run_reference(args):
    """--impl reference: the reference's CPU path = the oracle port (Taichi is not installable here)."""
    rank = int(os.environ.get("RANK", 0))
    if rank != 0:
        return 0
    name, sc = scene_for(args.gpus, args.scene)
    from oracle.sph_oracle import OracleSim
    o = OracleSim(sc)
    o.initialize()
    cores, table = best_thread_count(o)
    t0 = time.perf_counter()
    o.step()
    first = time.perf_counter() - t0
    budget = 150.0
    warm = max(1, min(args.warmup, int(0.2 * budget / max(first, 1e-6))))
    for _ in range(warm):
        o.step()
    k = max(1, min(args.steps, int(0.8 * budget / max(first, 1e-6))))
    t0 = time.perf_counter()
    for _ in range(k):
        o.step()
    dt = time.perf_counter() - t0
    val = k / dt
    line = {
        "impl": "reference", "metric": METRIC, "value": val * o.n / 1e6, "unit": UNIT, "steps_per_s": val,
        "n_gpus": args.gpus,
        "steps": k, "warmup": warm, "requested_steps": args.steps, "ms_per_step": 1e3 * dt / k,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(name, sc, o.n, int((o.material == 1).sum())),
        "cpu_baseline": {"value": val * o.n / 1e6, "unit": UNIT, "steps_per_s": val, "cores": cores, "kind": "port",
                         "threads_tried": {str(n_): round(v_, 2) for n_, v_ in table.items()},
                         "sample": f"{k} full steps of {name} ({o.n} particles); " + thread_note(cores, table)
                                   + " (OpenMP C restatement of the reference; Taichi cannot be installed offline)"},
        "e2e": {"value": val * o.n / 1e6, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))
    return 0


def pair_work(grid_ids, fluid_mask, grid_num, accepted_pairs):
    """Compute-side work of ONE pass over the neighbourhood (SURVEY.md section 8d): candidate distance
    tests = sum over fluid particles of the population of their 27-cell neighbourhood (cells outside the
    grid skipped, cell 0 invisible as in the reference), and the accepted pairs the lists hold."""
    import numpy as np
    gx, gy, gz = (int(v) for v in grid_num)
    cnt = np.bincount(grid_ids, minlength=gx * gy * gz).astype(np.int64)
    cnt[0] = 0  # particle_system.py:383: the range of cell 0 is empty
    c3 = cnt.reshape(gx, gy, gz)
    pad = np.zeros((gx + 2, gy + 2, gz + 2), np.int64)
    pad[1:-1, 1:-1, 1:-1] = c3
    nb = np.zeros_like(c3)
    for dx in range(3):
        for dy in range(3):
            for dz in range(3):
                nb += pad[dx:dx + gx, dy:dy + gy, dz:dz + gz]
    fluid_per_cell = np.bincount(grid_ids[fluid_mask], minlength=gx * gy * gz).astype(np.int64)
    tests = int((fluid_per_cell * nb.reshape(-1)).sum())
    return {"candidate_tests_per_pass": tests, "accepted_pairs_per_pass": int(accepted_pairs)}


def run_single(args):
    import torch
    from sph_taichi_b200 import ParticleSystem, SimConfig

    name, sc = scene_for(1, args.scene)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ps = ParticleSystem(SimConfig(sc), device=dev)
    solver = ps.build_solver()
    solver.initialize()
    eng = ps._engine
    n = ps.particle_max_num
    K, W = args.steps, args.warmup
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)  # > 50 MB L2

    solver.step(W)
    eng.check_status()
    torch.cuda.synchronize()

    # ---- value: K steps, L2 flushed between steps, CUDA events on the launching stream ----
    BAD = {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    for attempt in range(2):  # a run that saw a thermal / hw slowdown is rejected and re-measured once
        sampler = ClockSampler(0)
        solver.step(3)
        torch.cuda.synchronize()
        sampler.start()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
        launches0 = eng.launch_count()
        torch.cuda.synchronize()
        for a, b in ev:
            flush.zero_()
            a.record()
            solver.step()
            b.record()
        torch.cuda.synchronize()
        launches = eng.launch_count() - launches0
        cold_ms = sum(a.elapsed_time(b) for a, b in ev)
        if attempt == 0 and args.dump_outputs:  # the first window: W + 3 + K steps whether or not it is re-measured
            outputs = snapshot_outputs(ps)
        # ---- steady state: K back-to-back steps (state stays in L2, as in a real run) ----
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        solver.step(K)
        b.record()
        torch.cuda.synchronize()
        steady_ms = a.elapsed_time(b)
        clocks = sampler.stop()
        clocks["remeasured"] = attempt == 1
        if not (BAD & set(clocks.get("reasons", []))):
            break
    eng.check_status()

    # ---- per-kernel stage times (CUDA events between launches, un-graphed steps) ----
    stages = {}
    P = 20 if sc["Configuration"]["simulationMethod"] == 0 else 0  # the stage profiler covers the WCSPH step
    for _ in range(P):
        for k_, v_ in eng.profile_step().items():
            stages[k_] = stages.get(k_, 0.0) + v_ / P
    torch.cuda.synchronize()
    peak, peak_src = measured_hbm_peak()

    # ---- e2e: public surface, pinned host buffers, H2D + step + D2H every step ----
    hx = torch.empty((n, 3), dtype=torch.float32).pin_memory()
    hv = torch.empty((n, 3), dtype=torch.float32).pin_memory()
    ps.download_state(hx, hv)
    torch.cuda.synchronize()
    Ke = max(3, min(K, 100))
    # link diagnostic: the same pinned buffers, copies only (explains e2e on boxes with a slow PCIe path)
    dx = torch.empty_like(hx, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        dx.copy_(hx, non_blocking=True); hv.copy_(dx, non_blocking=True)
    torch.cuda.synchronize()
    link_gbs = 5 * 2 * hx.numel() * 4 / (time.perf_counter() - t0) / 1e9
    for _ in range(3):
        ps.upload_state(hx, hv); solver.step(); ps.download_state(hx, hv)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(Ke):
        ps.upload_state(hx, hv)
        solver.step()
        ps.download_state(hx, hv)
        torch.cuda.current_stream().synchronize()
    e2e_s = time.perf_counter() - t0
    eng.check_status()

    # ---- compute-side figure of the pair kernels (they are not HBM-bound; SURVEY.md section 8d) ----
    compute = None
    try:
        stats = eng.neighbor_stats()
        work = pair_work(ps.grid_ids.to_numpy(), ps.material.to_numpy() == 1, ps.grid_num, stats["pairs"])
        sps = K / (cold_ms * 1e-3)
        compute = dict(work, unit="per second, whole step (1 scan pass in the density kernel, 2 list passes)",
                       candidate_tests_per_s=work["candidate_tests_per_pass"] * sps,
                       interactions_per_s=2 * work["accepted_pairs_per_pass"] * sps,
                       mean_neighbours=stats["mean"], max_neighbours=stats["max"])
    except Exception as exc:  # diagnostics only: never lose the bench line over it
        compute = {"error": str(exc)[:200]}

    # ---- BASELINE cfg 3 in the same run (short leg; the driver only ever launches N = 1 with the default scene) ----
    extra = []
    if args.scene is None and os.environ.get("SPH_BENCH_SKIP_EXTRA") != "1":
        try:
            extra.append(extra_leg("armadillo_bath_dynamic", steps=20, warmup=10))
        except Exception as exc:  # never lose the main line over the extra leg
            extra.append({"workload": "armadillo_bath_dynamic", "error": str(exc)[:200]})

    cpu, _ = time_cpu_oracle(sc, budget_s=float(os.environ.get("SPH_BENCH_CPU_BUDGET_S", "15")))

    val = K / (cold_ms * 1e-3)
    total_ms = stages.get("total", 0.0)
    work = compute if compute and "error" not in compute else None
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    kernels = [roofline_entry(kind, name, n, stages.get(kind, 0.0), total_ms, peak, work, clocks.get("sm_mhz"), sms)
               for kind in ("density", "force") if stages.get(kind, 0.0) > 0]
    kernels.sort(key=lambda e: -e["avg_launch_ms"])
    roof = dict(kernels[0]) if kernels else {"bound": "hbm", "achieved": 0.0, "peak": peak, "unit": "GB/s", "frac": 0.0,
                                             "traffic": None}
    roof.update(peak_source=peak_src, kernels=kernels,
                whole_step={"algorithmic_bytes": 368 * n + 12 * int(ps.grid_num.prod()),
                            "achieved": (368 * n + 12 * int(ps.grid_num.prod())) / (cold_ms / K * 1e-3) / 1e9, "unit": "GB/s"},
                note="the top-level fields are the DOMINANT kernel of the step (largest CUDA-event time, un-graphed "
                     "sph_profile_step, 20 steps); `kernels` lists both pair kernels.  They are fp32-issue / L1 bound "
                     "(~80-100 flop/B), so the HBM fraction is small by construction; `compute_side` is the same launch "
                     "against the fp32 lane-op peak (DESIGN.md section 5)")
    line = {
        "metric": METRIC, "value": val * n / 1e6, "unit": UNIT, "steps_per_s": val, "n_gpus": 1, "steps": K,
        "warmup": W, "ms_per_step": cold_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "steady": {"value": K / (steady_ms * 1e-3) * n / 1e6, "unit": UNIT, "steps_per_s": K / (steady_ms * 1e-3),
                   "ms_per_step": steady_ms / K,
                   "note": "back-to-back CUDA-graph steps, state L2-resident (no flush)"},
        "readme_rtx3090_steps_per_s": 280.0 if name == "dragon_bath" else None,
        "config": workload_config(name, sc, n, ps.fluid_particle_num),
        "clocks": clocks,
        "e2e": {"value": Ke / e2e_s * n / 1e6, "unit": UNIT, "steps_per_s": Ke / e2e_s, "steps": Ke,
                "h2d_bytes_per_step": int(n * 24),
                "d2h_bytes_per_step": int(n * 24),
                "pinned_copy_gbs_this_box": round(link_gbs, 2),
                "note": "ParticleSystem.upload_state -> WCSPHSolver.step -> download_state, pinned host x and v; "
                        "link-bound: the two copies alone take 2 x 24 B x particles / the pinned-copy rate"},
        "gpu_launches": int(launches),
        "compute": compute,
        "roofline": roof,
        "stage_ms": {k_: round(v_, 5) for k_, v_ in stages.items()},
        "extra_configs": extra,
        "cpu_baseline": cpu,
    }
    if args.dump_outputs:
        write_outputs(args.dump_outputs, outputs)
    print(json.dumps(line))
    return 0


DUMP_FIELDS = ("x", "v", "density", "pressure", "x_0")
DUMP_MAX_BYTES = 64_000_000 - 64 * 1024  # 64 MB in all, with room for the .npy headers


def snapshot_outputs(ps):
    """The per-particle state a caller of solver.step() reads, as float32, rows ordered by (object_id, x_0): the
    engine's particle order is a detail of the neighbour sort, the rest position identifies a particle.  Above
    DUMP_MAX_BYTES a fixed seeded sample of the rows is kept."""
    import numpy as np
    x0, oid = ps.x_0.to_numpy(), ps.object_id.to_numpy()
    rows = np.lexsort((x0[:, 2], x0[:, 1], x0[:, 0], oid))
    out = {k: getattr(ps, k).to_numpy()[rows].astype(np.float32) for k in DUMP_FIELDS}
    row_bytes = sum(a[0].nbytes for a in out.values())
    if row_bytes * len(rows) > DUMP_MAX_BYTES:
        keep = np.sort(np.random.default_rng(0).choice(len(rows), DUMP_MAX_BYTES // row_bytes, replace=False))
        out = {k: a[keep] for k, a in out.items()}
    return out


def write_outputs(out_dir, arrays):
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, f"{name}.npy"), a)


def extra_leg(name, steps, warmup):
    """A short device-timed leg of another single-GPU BASELINE config (L2 flushed between steps, CUDA events)."""
    import torch
    from sph_taichi_b200 import ParticleSystem, SimConfig
    _, sc = scene_for(1, name)
    dev = torch.device("cuda:0")
    ps = ParticleSystem(SimConfig(sc), device=dev)
    solver = ps.build_solver()
    solver.initialize()
    solver.step(warmup)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for a, b in ev:
        flush.zero_()
        a.record()
        solver.step()
        b.record()
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in ev) / steps
    ps._engine.check_status()
    stages = {}
    for _ in range(5):
        for k_, v_ in ps._engine.profile_step().items():
            stages[k_] = stages.get(k_, 0.0) + v_ / 5
    n = ps.particle_max_num
    out = {"config": workload_config(name, sc, n, ps.fluid_particle_num), "steps": steps, "warmup": warmup,
           "ms_per_step": ms, "steps_per_s": 1e3 / ms, "value": 1e3 / ms * n / 1e6, "unit": UNIT,
           "readme_rtx3090_steps_per_s": 80.0 if name == "armadillo_bath_dynamic" else None,
           "stage_ms": {k_: round(v_, 5) for k_, v_ in stages.items()}}
    del solver, ps, flush
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--scene", default=None)
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the state after the last timed step as DIR/<name>.npy (single GPU)")
    args = ap.parse_args()
    multi = args.gpus > 1 or int(os.environ.get("WORLD_SIZE", "1")) > 1
    if args.dump_outputs and (multi or args.impl != "b200"):
        ap.error("--dump-outputs is implemented for the single-GPU run of the CUDA engine")
    if args.warmup < 3:
        args.warmup = 3
    if args.impl == "reference":
        if int(os.environ.get("RANK", 0)) == 0:
            pin_openmp_for_the_cpu_arm()
        return run_reference(args)
    if args.gpus == 1 and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        pin_openmp_for_the_cpu_arm()  # the cpu_baseline leg of the single-GPU line
    if args.gpus > 1 or int(os.environ.get("WORLD_SIZE", "1")) > 1:
        from sph_taichi_b200 import slab
        return slab.bench_main(args)
    return run_single(args)


if __name__ == "__main__":
    sys.exit(main())
