"""The mode of a sharded run: which requests ``slab.build_sharded`` refuses, with which exception and message, and how
many send layers an accepted one plans its slabs with; and the whole-scene start-up state it hands every rank.

The refusal table runs without a device: ``engine.Engine`` raises a sentinel, so an accepted request stops at its first
device work and a refused one must raise before it.  The start-up test runs on the device (or, with SPH_EMU_LIB, on
the host-emulated build of the library)."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 0.02
METHODS = (0, 2, 3, 4)
SCENES = ("fluid", "static block", "dynamic block", "dynamic body")


class _DeviceWork(Exception):
    pass


def _scene(kind, method=0):
    """A small dam break with ``kind``'s solid on its surface (none for "fluid"), run by ``method``."""
    from sph_taichi_b200 import scene
    sc = scene.dam_break_box([10, 6, 6], domain_end=[0.6, 0.4, 0.3], start=[0.06] * 3)
    sc["Configuration"]["simulationMethod"] = method
    top = 0.06 + 6 * D
    if kind in ("static block", "dynamic block"):
        sc["RigidBlocks"] = [{"objectId": 1, "start": [0.1, top, 0.08], "end": [0.15, top + 0.05, 0.13],
                              "translation": [0.0, 0.0, 0.0], "scale": [1, 1, 1], "velocity": [0.0, 0.0, 0.0],
                              "density": 600.0, "color": [255, 0, 0], "isDynamic": kind == "dynamic block"}]
    if kind == "dynamic body":
        sc["RigidBodies"] = [{"objectId": 2, "geometryFile": os.path.join(ROOT, "tests", "golden", "cube.obj"),
                              "translation": [0.2, top + 0.25 * D, 0.08], "rotationAxis": [0, 1, 0],
                              "rotationAngle": 0, "scale": [4.5 * D] * 3, "velocity": [0.0, 0.0, 0.0],
                              "density": 800.0, "color": [255, 255, 255], "isDynamic": True}]
    return sc


def _expected(method, kind, dynamic_solids, iisph, iisph_bodies):
    """(exception type, message) of a refused request, or the send-layer width of an accepted one."""
    from sph_taichi_b200 import slab
    dynamic = kind.startswith("dynamic")
    if iisph_bodies and method != 3:
        return ValueError, (f"iisph_bodies=True shards an IISPH scene (simulationMethod 3) with dynamic solids, not "
                            f"simulationMethod {method}")
    if method == 3 and not (iisph or iisph_bodies):
        return NotImplementedError, slab.IISPH_SINGLE_GPU
    if method not in (0, 3, 4):
        return NotImplementedError, (f"x-slab sharding runs WCSPH (0), DFSPH (4) and IISPH (3) scenes, not "
                                     f"simulationMethod {method}")
    if iisph and method != 3:
        return ValueError, f"iisph=True shards an IISPH scene (simulationMethod 3), not simulationMethod {method}"
    if iisph and not iisph_bodies and (dynamic_solids or dynamic):
        return NotImplementedError, slab.DYNAMIC_SOLIDS_IISPH
    bodies = dynamic_solids or iisph_bodies
    if bodies and method == 4:
        return NotImplementedError, slab.DYNAMIC_SOLIDS_WCSPH_ONLY
    if dynamic and not bodies:
        return NotImplementedError, slab.STATIC_SOLIDS_ONLY
    return slab.SEND_LAYERS_BODIES if bodies else slab.SEND_LAYERS


def test_build_sharded_mode_table(monkeypatch):
    """Every scene method, scene kind and opt-in flag: a refused request raises its exception and message before any
    device work; an accepted one plans its slabs with its mode's send layers (one more layer wide) and then reaches
    device work."""
    from sph_taichi_b200 import engine, slab

    def no_engine(*a, **k):
        raise _DeviceWork
    monkeypatch.setattr(engine, "Engine", no_engine)
    planned = []
    plan_slabs = slab.plan_slabs

    def spy(layer_counts, world, min_width=slab.SEND_LAYERS + 1):
        planned.append(min_width)
        return plan_slabs(layer_counts, world, min_width)
    monkeypatch.setattr(slab, "plan_slabs", spy)
    outcomes = {}
    for method in METHODS:
        for kind in SCENES:
            sc = _scene(kind, method)
            for flags in np.ndindex(2, 2, 2):
                dynamic_solids, iisph, iisph_bodies = (bool(f) for f in flags)
                want = _expected(method, kind, dynamic_solids, iisph, iisph_bodies)
                cell = (method, kind, dynamic_solids, iisph, iisph_bodies)
                planned.clear()
                with pytest.raises(Exception) as exc:
                    slab.build_sharded(sc, 0, 1, "cpu", dynamic_solids=dynamic_solids, iisph=iisph,
                                       iisph_bodies=iisph_bodies)
                if isinstance(want, tuple):
                    assert (exc.type, str(exc.value)) == want, cell
                    outcomes[want[0].__name__] = outcomes.get(want[0].__name__, 0) + 1
                else:
                    assert exc.type is _DeviceWork, (cell, exc.value)
                    assert planned == [want + 1], (cell, planned)
                    outcomes[want] = outcomes.get(want, 0) + 1
    # 128 cells.  Accepted without bodies: no opt-in on the fluid and static scenes in WCSPH and DFSPH, iisph=True
    # alone on them in IISPH.  With bodies: dynamic_solids=True alone in WCSPH (every scene), iisph_bodies=True with
    # any other flags in IISPH.
    assert outcomes == {slab.SEND_LAYERS: 6, slab.SEND_LAYERS_BODIES: 20, "ValueError": 64,
                        "NotImplementedError": 38}, outcomes


@pytest.mark.gpu
def test_startup_state_equals_the_single_engine(monkeypatch):
    """The start-up m_V of every solid (by solid id) and the bodies' rest centres of mass that ``build_sharded`` hands
    the ranks are bit-identical to what ``ParticleSystem`` + ``initialize()`` computes on the same scene: a static
    block, a shape-matched cube and a dynamic block around a dam break."""
    import torch
    from sph_taichi_b200 import ParticleSystem, SimConfig, slab

    sc = _scene("dynamic body")
    sc["RigidBlocks"] = _scene("static block")["RigidBlocks"] + [
        dict(_scene("dynamic block")["RigidBlocks"][0], objectId=3, start=[0.1, 0.24, 0.08], end=[0.15, 0.29, 0.13])]
    dev = torch.device("cpu" if os.environ.get("SPH_EMU_LIB") else "cuda:0")
    seen = {}
    select_owned = slab.select_owned

    def spy(arrays, h, lo, hi):  # build_sharded's whole-scene arrays, start-up m_V included
        seen["arrays"] = {k: np.array(v) for k, v in arrays.items()}
        return select_owned(arrays, h, lo, hi)
    monkeypatch.setattr(slab, "select_owned", spy)
    sim, _ = slab.build_sharded(sc, 0, 1, dev, dynamic_solids=True)
    arrays = seen["arrays"]
    sid = arrays["solid_id"]
    solid = sid >= 0
    mv_sharded = np.empty(int(solid.sum()), np.float32)
    mv_sharded[sid[solid]] = arrays["m_V"][solid]

    ps = ParticleSystem(SimConfig(sc), device=dev)
    ps.build_solver().initialize()
    ps._pull()
    n = int(ps.particle_num[None])
    sid1, mv1 = ps._t["solid_id"][:n].cpu().numpy(), ps._t["m_V"][:n].cpu().numpy()
    mv_single = np.empty(int((sid1 >= 0).sum()), np.float32)
    mv_single[sid1[sid1 >= 0]] = mv1[sid1 >= 0]
    assert mv_sharded.tobytes() == mv_single.tobytes()
    assert (arrays["m_V"][~solid] == np.float32(0.8 * D ** 3)).all()

    assert [b[0] for b in sim.bodies] == sorted(ps._body_index) == [2]
    for oid, _b0, _b1, rest_cm in sim.bodies:
        assert np.asarray(rest_cm, np.float32).tobytes() == np.asarray(ps.rigid_rest_cm[oid], np.float32).tobytes()
