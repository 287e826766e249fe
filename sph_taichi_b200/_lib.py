"""ctypes binding of ``libsph_b200.so`` (the C ABI in ``include/sph_b200.h``) and its build.

There is no CPU fallback: ``load()`` raises if the shared library is missing and
``Engine`` raises if no CUDA device can be used.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
LIB_PATH = os.environ.get("SPH_B200_LIB") or os.path.join(_PKG, "libsph_b200.so")  # override: experiments only
CSRC = os.path.join(_PKG, "csrc")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC", "-ldl"]

# every symbol include/sph_b200.h declares (tests check the .so exports all of them)
ABI_SYMBOLS = [
    "sph_workspace_bytes", "sph_create", "sph_destroy", "sph_last_error", "sph_set_params", "sph_set_solid_count", "sph_set_fluid_uniform",
    "sph_pack", "sph_unpack", "sph_unpack_xv", "sph_upload_xv", "sph_copy_grid_particles_num", "sph_neighbor_build",
    "sph_boundary_volume", "sph_compute_densities", "sph_compute_non_pressure_forces", "sph_compute_pressure_forces",
    "sph_advect", "sph_enforce_boundary", "sph_set_rigid_bodies", "sph_compute_com", "sph_compute_rigid_rest_cm",
    "sph_solve_constraints", "sph_get_rigid_state", "sph_step", "sph_read_status", "sph_clear_status", "sph_neighbor_stats", "sph_particle_count",
    "sph_launch_count", "sph_profile_step", "sph_timer_name", "sph_state_offsets", "sph_set_dfsph", "sph_dfsph_op", "sph_dfsph_solve", "sph_dfsph_step",
    "sph_comm_unique_id", "sph_comm_init_nccl", "sph_comm_set_transport", "sph_shard_configure", "sph_shard_begin",
    "sph_shard_step", "sph_halo_exchange", "sph_shard_info", "sph_shard_profile_step", "sph_shard_dfsph_step",
    "sph_shard_transport_stats", "sph_shard_configure_bodies", "sph_shard_dump", "sph_set_iisph", "sph_iisph_op",
    "sph_iisph_solve", "sph_iisph_step", "sph_iisph_read", "sph_shard_iisph_step", "sph_shard_configure_iisph_bodies",
    "sph_set_pcisph", "sph_pcisph_op", "sph_pcisph_solve", "sph_pcisph_step", "sph_pcisph_read",
    "sph_shard_configure_pcisph", "sph_shard_pcisph_step",
]


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))] + [
        os.path.join(_ROOT, "include", "sph_b200.h")]


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/sph_b200.cu for sm_90a (H100) into the in-tree shared library."""
    srcs = sources()
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return LIB_PATH
    nvcc = os.environ.get("NVCC") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB_PATH, os.path.join(CSRC, "sph_b200.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode:
        print(" ".join(cmd))
        print(res.stdout, res.stderr)
    if res.returncode:
        raise RuntimeError("nvcc failed building libsph_b200.so:\n" + res.stderr)
    return LIB_PATH


class SphParams(C.Structure):
    _fields_ = [("dim", C.c_int32), ("grid_num", C.c_int32 * 3), ("h", C.c_float), ("diameter", C.c_float),
                ("m_V0", C.c_float), ("density0", C.c_float), ("stiffness", C.c_float), ("exponent", C.c_float),
                ("viscosity", C.c_float), ("surface_tension", C.c_float), ("dt", C.c_float), ("g", C.c_float * 3),
                ("domain_size", C.c_float * 3), ("k_w", C.c_float), ("k_dw", C.c_float), ("visc_eps", C.c_float),
                ("clamp_hi", C.c_float * 3)]


class SphFields(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in (
        "object_id", "x", "x_0", "v", "acceleration", "m_V", "m", "density", "pressure", "material", "is_dynamic",
        "color", "grid_ids", "solid_id", "dfsph_factor", "density_adv")]


# halo-exchange transport (include/sph_b200.h: SphTransport); the CPU test-suite fills it with gloo callbacks
TRANSPORT_GROUP_START = C.CFUNCTYPE(C.c_int, C.c_void_p)
TRANSPORT_GROUP_END = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)
TRANSPORT_SEND = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p)
TRANSPORT_RECV = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p)


class SphTransport(C.Structure):
    _fields_ = [("user", C.c_void_p), ("group_start", TRANSPORT_GROUP_START), ("group_end", TRANSPORT_GROUP_END),
                ("send", TRANSPORT_SEND), ("recv", TRANSPORT_RECV)]


class SphRigidBody(C.Structure):
    _fields_ = [("object_id", C.c_int32), ("solid_begin", C.c_int32), ("solid_end", C.c_int32),
                ("rest_cm", C.c_float * 3)]


class SphDfsphStep(C.Structure):
    _fields_ = [("enable_divergence_solver", C.c_int32), ("max_iterations_v", C.c_int32), ("max_iterations", C.c_int32),
                ("eta_v", C.c_double), ("eta", C.c_double), ("inv_dt", C.c_float), ("dt", C.c_float),
                ("inv_dt2", C.c_float), ("density0", C.c_float), ("n_fluid", C.c_int64),
                ("first_batch_v", C.c_int32), ("first_batch", C.c_int32), ("iterations_v", C.c_int32),
                ("iterations", C.c_int32), ("avg_err_v", C.c_double), ("avg_err", C.c_double)]


class SphIisphStep(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("omega", C.c_float), ("eta", C.c_double), ("n_fluid", C.c_int64),
                ("first_batch", C.c_int32), ("iterations", C.c_int32), ("avg_err", C.c_double)]


class SphPcisphStep(C.Structure):
    _fields_ = [("delta", C.c_float), ("eta", C.c_double), ("min_iterations", C.c_int32), ("max_iterations", C.c_int32),
                ("first_batch", C.c_int32), ("iterations", C.c_int32), ("max_err", C.c_double)]


_lib = None


def load():
    """Load the shared library (no auto-build on a machine without nvcc; fails loudly)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        try:
            build()
        except Exception as exc:  # pragma: no cover - depends on toolchain
            raise RuntimeError(
                f"{LIB_PATH} is missing and could not be built ({exc}); the CUDA engine is required "
                "(there is no CPU fallback). Run `python -c 'import __graft_entry__ as g; g.build()'`.") from exc
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
    PP = C.POINTER(SphParams)
    FP = C.POINTER(SphFields)
    sig = {
        "sph_workspace_bytes": (u64, [PP, i64, i64, i32]),
        "sph_create": (C.c_int, [PP, i64, i64, i32, i32, vp, u64, C.POINTER(vp)]),
        "sph_destroy": (C.c_int, [vp]),
        "sph_last_error": (C.c_char_p, [vp]),
        "sph_set_params": (C.c_int, [vp, PP]),
        "sph_set_solid_count": (C.c_int, [vp, i64, i32]),
        "sph_set_fluid_uniform": (C.c_int, [vp, i32, C.c_float, C.c_float]),
        "sph_pack": (C.c_int, [vp, FP, i64, vp]),
        "sph_unpack": (C.c_int, [vp, FP, vp]),
        "sph_unpack_xv": (C.c_int, [vp, vp, vp, vp, vp]),
        "sph_upload_xv": (C.c_int, [vp, vp, vp, vp]),
        "sph_copy_grid_particles_num": (C.c_int, [vp, vp, vp]),
        "sph_neighbor_build": (C.c_int, [vp, vp]),
        "sph_boundary_volume": (C.c_int, [vp, i32, vp]),
        "sph_compute_densities": (C.c_int, [vp, vp]),
        "sph_compute_non_pressure_forces": (C.c_int, [vp, vp]),
        "sph_compute_pressure_forces": (C.c_int, [vp, vp]),
        "sph_advect": (C.c_int, [vp, vp]),
        "sph_enforce_boundary": (C.c_int, [vp, i32, vp]),
        "sph_set_rigid_bodies": (C.c_int, [vp, C.POINTER(SphRigidBody), i32]),
        "sph_compute_com": (C.c_int, [vp, i32, vp, vp]),
        "sph_compute_rigid_rest_cm": (C.c_int, [vp, i32, vp]),
        "sph_solve_constraints": (C.c_int, [vp, i32, vp, vp]),
        "sph_get_rigid_state": (C.c_int, [vp, i32, vp, vp]),
        "sph_step": (C.c_int, [vp, i32, vp]),
        "sph_read_status": (C.c_int, [vp, C.POINTER(C.c_uint32), vp]),
        "sph_clear_status": (C.c_int, [vp, vp]),
        "sph_neighbor_stats": (C.c_int, [vp, vp, vp]),
        "sph_particle_count": (i64, [vp]),
        "sph_launch_count": (i64, [vp]),
        "sph_profile_step": (C.c_int, [vp, C.POINTER(C.c_float), i32, vp]),
        "sph_timer_name": (C.c_char_p, [i32]),
        "sph_state_offsets": (C.c_int, [vp, C.POINTER(u64)]),
        "sph_set_dfsph": (C.c_int, [vp, i32]),
        "sph_dfsph_op": (C.c_int, [vp, i32, C.c_float, vp, vp]),
        "sph_dfsph_solve": (C.c_int, [vp, i32, i32, C.c_double, C.c_float, i64, i32, C.POINTER(i32), C.POINTER(i32),
                                      C.POINTER(C.c_double), vp]),
        "sph_dfsph_step": (C.c_int, [vp, i32, C.POINTER(SphDfsphStep), vp]),
        "sph_comm_unique_id": (C.c_int, [C.c_char_p]),
        "sph_comm_init_nccl": (C.c_int, [vp, C.c_char_p, i32, i32]),
        "sph_comm_set_transport": (C.c_int, [vp, C.POINTER(SphTransport), i32, i32]),
        "sph_shard_configure": (C.c_int, [vp, i32, i32, i32, i64, i32]),
        "sph_shard_configure_bodies": (C.c_int, [vp, i32, i32, i32, i64, i32, C.POINTER(SphRigidBody), i32]),
        "sph_shard_configure_iisph_bodies": (C.c_int, [vp, i32, i32, i32, i64, i32, C.POINTER(SphRigidBody), i32]),
        "sph_shard_begin": (C.c_int, [vp, vp]),
        "sph_shard_step": (C.c_int, [vp, i32, vp]),
        "sph_halo_exchange": (C.c_int, [vp, vp]),
        "sph_shard_info": (C.c_int, [vp, C.POINTER(i32), C.POINTER(u64), vp]),
        "sph_shard_profile_step": (C.c_int, [vp, C.POINTER(C.c_float), vp]),
        "sph_shard_dfsph_step": (C.c_int, [vp, i32, C.POINTER(SphDfsphStep), vp]),
        "sph_shard_transport_stats": (C.c_int, [vp, C.POINTER(u64)]),
        "sph_shard_dump": (C.c_int, [vp, i32, vp, vp, i64, C.POINTER(i64), C.POINTER(C.c_uint32), vp]),
        "sph_set_iisph": (C.c_int, [vp, i32]),
        "sph_iisph_op": (C.c_int, [vp, i32, C.c_float, vp, vp]),
        "sph_iisph_solve": (C.c_int, [vp, i32, C.c_float, C.c_double, i64, i32, C.POINTER(i32), C.POINTER(C.c_double),
                                      vp]),
        "sph_iisph_step": (C.c_int, [vp, i32, C.POINTER(SphIisphStep), vp]),
        "sph_iisph_read": (C.c_int, [vp, vp, vp, vp, vp]),
        "sph_shard_iisph_step": (C.c_int, [vp, i32, C.POINTER(SphIisphStep), vp]),
        "sph_set_pcisph": (C.c_int, [vp, i32]),
        "sph_pcisph_op": (C.c_int, [vp, i32, C.c_float, vp, vp]),
        "sph_pcisph_solve": (C.c_int, [vp, C.c_float, C.c_double, i32, i32, i32, C.POINTER(i32), C.POINTER(C.c_double),
                                       vp]),
        "sph_pcisph_step": (C.c_int, [vp, i32, C.POINTER(SphPcisphStep), vp]),
        "sph_pcisph_read": (C.c_int, [vp, vp, vp, vp, vp]),
        "sph_shard_configure_pcisph": (C.c_int, [vp, i32, i32, i32, i64, i32]),
        "sph_shard_pcisph_step": (C.c_int, [vp, i32, C.POINTER(SphPcisphStep), vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
