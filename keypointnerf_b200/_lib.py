"""ctypes binding of the C ABI in include/kpnerf_b200.h (the product's only compute path).

There is no CPU fallback: if the shared library is missing this module raises, and
``kpn_create`` fails without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# KPN_LIB selects an alternative build of the same ABI (e.g. one built with extra -D flags for an experiment)
LIB_PATH = os.environ.get("KPN_LIB") or os.path.join(_HERE, "lib", "libkpnerf_b200.so")

KPN_OK = 0
KPN_MEM_DEVICE = 0
KPN_MEM_HOST = 1
KPN_NUM_LAYERS = 19
KPN_NHWC_FEAT64, KPN_NHWC_FEAT8, KPN_NHWC_FEATTEX = 1, 2, 4

EXPORTS = ["kpn_abi_version", "kpn_create", "kpn_destroy", "kpn_last_error", "kpn_set_weights", "kpn_set_scene",
           "kpn_render", "kpn_query", "kpn_get_stats", "kpn_set_profiling", "kpn_selftest_umma", "kpn_selftest_umma2", "kpn_debug_timing", "kpn_debug_kmap", "kpn_check_health", "kpn_reserve", "kpn_debug_stage_times", "kpn_decode_views",
           "kpn_query_grid", "kpn_mesh_begin", "kpn_mesh_emit", "kpn_render_rays", "kpn_camera_rays", "kpn_render_rays_backward"]
KPN_ABI_VERSION = 5

c_float_p = C.POINTER(C.c_float)
c_u8_p = C.POINTER(C.c_uint8)


class KpnLayer(C.Structure):
    _fields_ = [("w", C.c_void_p), ("g", C.c_void_p), ("bias", C.c_void_p), ("n_out", C.c_int), ("n_in", C.c_int)]


class KpnWeights(C.Structure):
    _fields_ = [("layer", KpnLayer * KPN_NUM_LAYERS), ("ani_al", C.c_float), ("n_kpt", C.c_int),
                ("sp_level", C.c_int), ("sp_scale", C.c_float), ("sp_sigma", C.c_float)]


class KpnScene(C.Structure):
    _fields_ = [("n_views", C.c_int), ("n_kpt", C.c_int),
                ("src_width", C.c_float), ("src_height", C.c_float),
                ("znear", C.c_float), ("zfar", C.c_float), ("nml_scale", C.c_float),
                ("KRT", C.c_void_p), ("extrin", C.c_void_p), ("kpt3d", C.c_void_p), ("bounds", C.c_void_p),
                ("feat64", C.c_void_p), ("f64_c", C.c_int), ("f64_h", C.c_int), ("f64_w", C.c_int),
                ("feat8", C.c_void_p), ("f8_c", C.c_int), ("f8_h", C.c_int), ("f8_w", C.c_int),
                ("feat_tex", C.c_void_p), ("ftex_c", C.c_int), ("ftex_h", C.c_int), ("ftex_w", C.c_int),
                ("img", C.c_void_p), ("img_h", C.c_int), ("img_w", C.c_int),
                ("fg", C.c_void_p), ("fg_h", C.c_int), ("fg_w", C.c_int),
                ("mem", C.c_int), ("layout", C.c_int)]


class KpnTarget(C.Structure):
    _fields_ = [("K", C.c_void_p), ("RT", C.c_void_p), ("znear", C.c_float), ("zfar", C.c_float),
                ("x0", C.c_int), ("y0", C.c_int), ("step", C.c_int), ("nx", C.c_int), ("ny", C.c_int),
                ("mem", C.c_int), ("step_y", C.c_int)]


class KpnOpts(C.Structure):
    _fields_ = [("sample_per_ray_c", C.c_int), ("sample_per_ray_f", C.c_int), ("fine", C.c_int),
                ("ert_eps", C.c_float), ("z_fine_override", C.c_void_p), ("engine", C.c_int)]


class KpnOut(C.Structure):
    _fields_ = [("tex_fg", C.c_void_p), ("depth", C.c_void_p), ("alpha", C.c_void_p),
                ("tex_fg_fine", C.c_void_p), ("depth_fine", C.c_void_p), ("alpha_fine", C.c_void_p),
                ("sdf", C.c_void_p), ("z_fine", C.c_void_p), ("contrib", C.c_void_p), ("mem", C.c_int)]


class KpnRays(C.Structure):
    _fields_ = [("origins", C.c_void_p), ("dirs", C.c_void_p), ("near_far", C.c_void_p), ("n", C.c_longlong), ("mem", C.c_int)]


class KpnGrads(C.Structure):
    _fields_ = [("dW", C.c_void_p * KPN_NUM_LAYERS), ("db", C.c_void_p * KPN_NUM_LAYERS), ("d_ani_al", C.c_void_p),
                ("d_feat64", C.c_void_p), ("d_feat8", C.c_void_p), ("d_feat_tex", C.c_void_p), ("mem", C.c_int)]


class KpnGrid(C.Structure):
    _fields_ = [("origin", C.c_float * 3), ("spacing", C.c_float * 3), ("nx", C.c_int), ("ny", C.c_int), ("nz", C.c_int)]


class KpnStats(C.Structure):
    _fields_ = [("samples_total", C.c_uint64), ("samples_valid", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("shade_launches", C.c_uint64), ("shade_ms", C.c_double), ("samples_coloured", C.c_uint64),
                ("geo_ms", C.c_double)]


_lib = None


def load() -> C.CDLL:
    """Load the shared library (built in-tree by ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "keypointnerf_b200 has no CPU or PyTorch fallback for the ray-march path.")
    lib = C.CDLL(LIB_PATH)
    lib.kpn_abi_version.restype = C.c_int
    if lib.kpn_abi_version() != KPN_ABI_VERSION:
        raise RuntimeError(f"{LIB_PATH} has ABI version {lib.kpn_abi_version()}, this binding expects {KPN_ABI_VERSION}: rebuild it")
    lib.kpn_check_health.argtypes = [C.c_void_p, C.c_void_p]
    lib.kpn_check_health.restype = C.c_int
    lib.kpn_reserve.argtypes = [C.c_void_p, C.c_longlong, C.c_int]
    lib.kpn_reserve.restype = C.c_int
    lib.kpn_decode_views.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_void_p]
    lib.kpn_decode_views.restype = C.c_int
    lib.kpn_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    lib.kpn_create.restype = C.c_int
    lib.kpn_destroy.argtypes = [C.c_void_p]
    lib.kpn_destroy.restype = None
    lib.kpn_last_error.argtypes = [C.c_void_p]
    lib.kpn_last_error.restype = C.c_char_p
    lib.kpn_set_weights.argtypes = [C.c_void_p, C.POINTER(KpnWeights)]
    lib.kpn_set_weights.restype = C.c_int
    lib.kpn_set_scene.argtypes = [C.c_void_p, C.POINTER(KpnScene), C.c_void_p]
    lib.kpn_set_scene.restype = C.c_int
    lib.kpn_render.argtypes = [C.c_void_p, C.POINTER(KpnTarget), C.POINTER(KpnOpts), C.POINTER(KpnOut), C.c_void_p]
    lib.kpn_render.restype = C.c_int
    lib.kpn_render_rays.argtypes = [C.c_void_p, C.POINTER(KpnRays), C.POINTER(KpnOpts), C.POINTER(KpnOut), C.c_void_p]
    lib.kpn_render_rays.restype = C.c_int
    lib.kpn_render_rays_backward.argtypes = [C.c_void_p, C.POINTER(KpnRays), C.POINTER(KpnOpts), C.POINTER(KpnOut),
                                             C.POINTER(KpnGrads), C.c_void_p]
    lib.kpn_render_rays_backward.restype = C.c_int
    lib.kpn_camera_rays.argtypes = [C.c_void_p, C.POINTER(KpnTarget), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.kpn_camera_rays.restype = C.c_int
    lib.kpn_query.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                              C.POINTER(KpnOpts), C.c_void_p]
    lib.kpn_query.restype = C.c_int
    lib.kpn_query_grid.argtypes = [C.c_void_p, C.POINTER(KpnGrid), C.c_void_p, C.c_void_p, C.c_int, C.POINTER(KpnOpts), C.c_void_p]
    lib.kpn_query_grid.restype = C.c_int
    lib.kpn_mesh_begin.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_longlong),
                                   C.c_void_p]
    lib.kpn_mesh_begin.restype = C.c_int
    lib.kpn_mesh_emit.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int, C.c_void_p]
    lib.kpn_mesh_emit.restype = C.c_int
    lib.kpn_get_stats.argtypes = [C.c_void_p, C.POINTER(KpnStats), C.c_void_p]
    lib.kpn_get_stats.restype = C.c_int
    lib.kpn_set_profiling.argtypes = [C.c_void_p, C.c_int]
    lib.kpn_set_profiling.restype = C.c_int
    lib.kpn_debug_timing.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.kpn_debug_timing.restype = C.c_int
    lib.kpn_debug_kmap.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.kpn_debug_kmap.restype = C.c_int
    lib.kpn_selftest_umma2.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.kpn_selftest_umma2.restype = C.c_int
    lib.kpn_selftest_umma.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.kpn_selftest_umma.restype = C.c_int
    _lib = lib
    return lib


class KpnError(RuntimeError):
    pass


def check(lib, ctx, rc: int, what: str):
    if rc != KPN_OK:
        msg = lib.kpn_last_error(ctx).decode() if ctx else ""
        raise KpnError(f"{what} failed with status {rc}: {msg}")
