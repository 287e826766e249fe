"""The CPU oracle against golden vectors produced by the REFERENCE'S OWN SOURCE.

tests/golden/ref_*.npz were written by tests/golden/make_reference_golden.py: erizmr/SPH_Taichi's unmodified
particle_system.py / sph_base.py / WCSPH.py / DFSPH.py executed under a pure-Python stand-in for the Taichi runtime
(serial loops, IEEE float32).  The oracle replays the same scenes; integer / ordering data must be identical,
float fields agree to a few float32 ulp of the field's scale (the stand-in evaluates constant sub-expressions in
double where Taichi folds them in float32, and the oracle multiplies by reciprocals in places)."""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
NAMES = sorted(f[4:-4] for f in os.listdir(GOLD) if f.startswith("ref_") and f.endswith(".npz") and "_body" not in f)
REL = 2e-5  # of the field's max magnitude, the tolerance of the GPU parity tests


def _close(a, b, rel=REL, what=""):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    scale = max(float(np.abs(b).max()), 1e-30)
    err = float(np.abs(a - b).max()) / scale
    assert err < rel, f"{what}: max rel err {err:.3e} (scale {scale:.3e})"


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_the_reference_source(name):
    from oracle.sph_oracle import OracleSim
    z = np.load(os.path.join(GOLD, f"ref_{name}.npz"))
    scene = json.loads(str(z["scene"]))
    for b in scene.get("RigidBodies", []):
        b["voxelizedPointsFile"] = os.path.join(GOLD, b["voxelizedPointsFile"])
    steps = int(z["steps"])
    o = OracleSim(scene)
    o.initialize()
    dfsph = scene["Configuration"]["simulationMethod"] == 4
    for stage in ("init_", "final_"):
        if stage == "final_":
            its = []
            for _ in range(steps):
                o.step()
                if dfsph:
                    its.append((o.last_iterations_v, o.last_iterations))
            if dfsph:  # the host-side convergence loops stop after the same number of sweeps
                assert [a for a, _ in its] == list(z["dfsph_iterations_v"]), (its, z["dfsph_iterations_v"])
                assert [b for _, b in its] == list(z["dfsph_iterations"]), (its, z["dfsph_iterations"])
        if stage + "x" not in z.files:  # the 8 K cube keeps the final state only (file size)
            continue
        # the reference's own particle order and integer data: exact
        for f in ("object_id", "material", "is_dynamic", "grid_ids", "grid_particles_num", "x_0"):
            if stage + f in z.files:
                assert np.array_equal(getattr(o, f), z[stage + f]), (stage, f)
        for f in ("x", "v", "m_V", "m", "density", "pressure", "acceleration"):
            if stage + f in z.files:
                _close(getattr(o, f), z[stage + f], what=f"{name} {stage}{f}")
        if dfsph:
            fl = o.material == 1
            _close(o.dfsph_factor[fl], z[stage + "dfsph_factor"][fl], 1e-4, f"{name} {stage}dfsph_factor")
            _close(o.density_adv[fl], z[stage + "density_adv"][fl], what=f"{name} {stage}density_adv")
    assert steps >= 3 and len(o.x) > 200 and "final_x" in z.files


def test_reference_goldens_cover_both_solvers_and_rigid_bodies():
    assert {"wcsph_blocks", "wcsph_walls", "wcsph_bodies", "wcsph_dambreak", "dfsph_blocks"} <= set(NAMES)
    # SURVEY Q3, observed when the vectors were made: upper-wall contacts read neighbour cells outside the grid
    assert int(np.load(os.path.join(GOLD, "ref_wcsph_walls.npz"))["oob_cell_reads"]) > 0

