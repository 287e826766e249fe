"""Host logic of bench.py that the GPU box cannot be asked about twice: the CPU arm's thread probe, the roofline
arithmetic, the candidate-test count, the workload description both arms must share."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


class _FakeOracle:
    """step() takes cost[threads] seconds of virtual time (perf_counter is patched)."""

    def __init__(self, cost, clock):
        self.cost, self.clock, self.threads, self.steps = cost, clock, None, []

    def step(self):
        self.clock[0] += self.cost[self.threads]
        self.steps.append(self.threads)


def _probe(monkeypatch, total, cost):
    import oracle.sph_oracle as so
    clock = [0.0]
    o = _FakeOracle(cost, clock)
    monkeypatch.setattr(so, "set_threads", lambda n: setattr(o, "threads", n))
    monkeypatch.setattr(bench.time, "perf_counter", lambda: clock[0])
    monkeypatch.setattr(bench.os, "cpu_count", lambda: total)
    monkeypatch.setattr(bench, "cgroup_cpu_quota", lambda: None)
    best, table = bench.best_thread_count(o, reps=3)
    return best, table, o


def test_thread_probe_stops_at_the_first_oversubscribed_count(monkeypatch):
    # a host with 128 hardware threads visible of which only 16-32 are scheduled
    best, table, o = _probe(monkeypatch, 128, {16: 0.070, 32: 0.072, 64: 0.16, 128: 1.4})
    assert best == 16 and set(table) == {16, 32, 64}      # 64 is abandoned after ONE step, 128 is never tried
    assert o.steps.count(64) == 1 and 128 not in o.steps and o.steps.count(16) == 4
    assert o.threads == 16                                 # the oracle is left at the chosen count


def test_thread_probe_goes_all_the_way_up_on_a_box_that_scales(monkeypatch):
    best, table, _ = _probe(monkeypatch, 8, {1: 1.0, 2: 0.52, 4: 0.27, 8: 0.15})
    assert best == 8 and set(table) == {1, 2, 4, 8}
    assert abs(table[8] - 1 / 0.15) < 1e-9


def test_roofline_entry_arithmetic():
    n, ms = 441_996, 0.1
    e = bench.roofline_entry("density", "no_such_workload", n, ms, 0.2, 6567.1,
                             {"candidate_tests_per_pass": 85_000_000, "accepted_pairs_per_pass": 10_800_000}, 1965.0, 132)
    assert abs(e["achieved"] - 24 * n / 1e-4 / 1e9) < 1e-9 and abs(e["frac"] - e["achieved"] / 6567.1) < 1e-12
    assert e["share_of_step"] == 0.5 and e["traffic"] is None and e["bound"] == "hbm"
    ops = 85_000_000 * 7 + 10_800_000 * 30
    cs = e["compute_side"]
    assert cs["fp32_lane_ops_per_launch"] == ops
    assert abs(cs["frac"] - ops / 1e-4 / (132 * 128 * 1965.0e6)) < 1e-12
    f = bench.roofline_entry("force", "no_such_workload", n, ms, 0.2, 6567.1,
                             {"candidate_tests_per_pass": 1, "accepted_pairs_per_pass": 10}, 1000.0, 114)
    assert f["algorithmic_bytes_per_particle"] == 52 and f["compute_side"]["fp32_lane_ops_per_launch"] == 540
    assert abs(f["compute_side"]["peak_lane_ops_per_s"] - 114 * 128 * 1000.0e6) < 1 and "114 SMs" in f["compute_side"]["formula"]


def test_candidate_test_count_against_brute_force():
    rng = np.random.default_rng(5)
    g = (4, 5, 3)
    ids = rng.integers(0, g[0] * g[1] * g[2], size=200)
    fluid = rng.random(200) < 0.7
    want = 0
    cnt = np.bincount(ids, minlength=60)
    cnt[0] = 0                                                  # cell 0 is invisible (particle_system.py:383)
    for c in ids[fluid]:
        i, j, k = c // 15, (c // 3) % 5, c % 3
        for a in (-1, 0, 1):
            for b in (-1, 0, 1):
                for d in (-1, 0, 1):
                    ii, jj, kk = i + a, j + b, k + d
                    if 0 <= ii < 4 and 0 <= jj < 5 and 0 <= kk < 3:
                        want += cnt[(ii * 5 + jj) * 3 + kk]
    got = bench.pair_work(ids, fluid, g, accepted_pairs=17)
    assert got == {"candidate_tests_per_pass": int(want), "accepted_pairs_per_pass": 17}


def test_both_arms_describe_the_same_workload():
    for n in (1, 2, 4, 8):
        name, sc = bench.scene_for(n)
        a = bench.workload_config(name, sc, 10, 7)
        b = bench.workload_config(name, sc, 10, 7)
        assert a == b and a["workload"] == {1: "dragon_bath", 2: "box_4m", 4: "box_4m", 8: "box_16m"}[n]
        assert a["solver"] == "WCSPH" and a["dt"] == 4e-4
    assert bench.workload_config(*bench.scene_for(1), 441_996, 423_500)["grid_cells"] == 468_750
