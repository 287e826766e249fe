"""Cost of the output path of a sharded run on one GPU: ``ShardedSimulation.dump(0)`` (synchronising, so a host clock
around it is a valid time) and ``run_simulation.write_ply_ascii`` of the same frame, on world-1 dragon_bath after
``--steps`` steps.  Prints one JSON line with the card name and its power limit.

    python tools/shard_export_timing.py [--scene dragon_bath] [--steps 40] [--repeat 5]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from run_simulation import write_ply_ascii  # noqa: E402
from sph_taichi_b200 import scene, slab  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="dragon_bath", choices=sorted(scene.NAMED_SCENES))
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    sim, n_total = slab.build_sharded(scene.NAMED_SCENES[a.scene](), 0, 1, dev)
    sim.step(a.steps)
    sim.dump(0)  # first call: allocates the buffers
    dump_ms = []
    for _ in range(a.repeat):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        out = sim.dump(0)
        dump_ms.append((time.perf_counter() - t0) * 1e3)
    ply_ms = []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            write_ply_ascii(os.path.join(tmp, "frame.ply"), out["position"])
            ply_ms.append((time.perf_counter() - t0) * 1e3)
    card, plimit = slab._gpu_name_and_power_limit(0)
    print(json.dumps({"scene": a.scene, "particles": int(n_total), "rows": int(out["position"].shape[0]),
                      "steps_before": a.steps, "dump_ms": dump_ms, "write_ply_ascii_ms": ply_ms,
                      "gpu": {"name": card, "power_limit_w": plimit}}))


if __name__ == "__main__":
    main()
