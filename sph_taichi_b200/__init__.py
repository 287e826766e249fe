"""sph_taichi_b200: a Hopper-native (sm_90a) WCSPH step engine behind the
ParticleSystem / SPHBase.step() surface of erizmr/SPH_Taichi."""
from .config_builder import SimConfig  # noqa: F401

__all__ = ["SimConfig", "ParticleSystem", "WCSPHSolver", "SPHBase"]


def __getattr__(name):
    # torch-dependent modules are imported lazily so that host-only tools stay light
    if name == "ParticleSystem":
        from .particle_system import ParticleSystem
        return ParticleSystem
    if name == "WCSPHSolver":
        from .WCSPH import WCSPHSolver
        return WCSPHSolver
    if name == "SPHBase":
        from .sph_base import SPHBase
        return SPHBase
    raise AttributeError(name)
