"""ctypes binding of the C ABI in include/gsplat_b200.h (pf3plat_b200/csrc/libgsplat_b200.so).

This is the only place the shared library is loaded.  There is NO fallback: if the library is missing or
was built for another ABI version the import fails loudly (the product path never routes through the CPU
oracle or any PyTorch re-implementation).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_uint32, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libgsplat_b200.so")
ABI_VERSION = 1

GS_FLAG_DEPTH = 1
GS_FLAG_PREFILTERED = 2
GS_TUNE_FORCE_RADIX_BINNING = 1
GS_TUNE_NO_SPECULATION = 2
GS_TUNE_SEPARATE_EMIT = 4
GS_TUNE_NO_STRATA = 8
GS_TUNE_BWD_V1 = 16
GS_TUNE_FWD_WS = 32
GS_TUNE_STRATA_MERGE_SORT = 64
GS_TUNE_BWD_OCC4 = 128
GS_TUNE_PRE_OCC6 = 4096
GS_TUNE_PBWD_2PHASE = 8192
GS_TUNE_NO_TILE_STRATA = 16384
GS_TUNE_DIRECT_OUTPUT = 32768
GS_TUNE_PRE_SH_RAW16 = 65536
GS_TUNE_NO_ZERO_COPY = 131072
GS_TUNE_NO_SPLIT_COLOUR = 262144
GS_TUNE_FEED_PIECES_SHIFT = 8
GS_NUM_STAGES = 8
STAGE_NAMES = ("preprocess", "bin_scan", "bin_emit", "bin_sort", "composite", "composite_bwd", "preprocess_bwd", "sh_colour")


class GsConfig(Structure):
    _fields_ = [
        ("P", c_int32), ("S", c_int32), ("V", c_int32), ("M", c_int32), ("sh_degree", c_int32),
        ("image_height", c_int32), ("image_width", c_int32), ("flags", c_uint32),
        ("tanfovx", c_float), ("tanfovy", c_float), ("scale_modifier", c_float),
        ("near_cull_z", c_float), ("dilation", c_float), ("guard_band", c_float),
        ("sh_eval_max_degree", c_int32), ("tuning", c_uint32),
        ("viewmatrix", c_void_p), ("projmatrix", c_void_p), ("campos", c_void_p), ("bg", c_void_p),
        ("tanfov", c_void_p), ("view_scale", c_void_p),
    ]


class GsInputs(Structure):
    _fields_ = [("means3D", c_void_p), ("opacities", c_void_p), ("shs", c_void_p), ("colors_precomp", c_void_p),
                ("scales", c_void_p), ("rotations", c_void_p), ("cov3D_precomp", c_void_p)]


class GsOutputs(Structure):
    _fields_ = [("color", c_void_p), ("radii", c_void_p), ("depth", c_void_p)]


class GsOutGrads(Structure):
    _fields_ = [("dL_dcolor", c_void_p), ("dL_ddepth", c_void_p)]


class GsInGrads(Structure):
    _fields_ = [("dL_dmeans3D", c_void_p), ("dL_dmeans2D", c_void_p), ("dL_dshs", c_void_p), ("dL_dcolors", c_void_p),
                ("dL_dopacities", c_void_p), ("dL_dscales", c_void_p), ("dL_drotations", c_void_p),
                ("dL_dcov3D", c_void_p)]


class GsStats(Structure):
    _fields_ = [("num_rendered", c_int64), ("num_visible", c_int64), ("saved_bytes", c_int64),
                ("scratch_bytes", c_int64), ("kernel_launches", c_int32), ("max_tile_list", c_int32),
                ("speculative", c_int32), ("overflow_redos", c_int32), ("pool_reserved_bytes", c_int64),
                ("pool_used_bytes", c_int64)]


# every symbol include/gsplat_b200.h declares: name -> (restype, argtypes)
class GsAdapterConfig(Structure):
    _fields_ = [("V", c_int32), ("R", c_int32), ("d_sh", c_int32), ("reserved_", c_int32),
                ("scale_min", c_float), ("scale_max", c_float), ("eps", c_float), ("reserved2_", c_float),
                ("c2w", c_void_p), ("kinv", c_void_p), ("multiplier", c_void_p), ("sh_rotation", c_void_p),
                ("sh_mask", c_void_p)]


class GsAdapterInputs(Structure):
    _fields_ = [("coordinates", c_void_p), ("depths", c_void_p), ("raw_gaussians", c_void_p)]


class GsAdapterOutputs(Structure):
    _fields_ = [("means", c_void_p), ("covariances", c_void_p), ("harmonics", c_void_p), ("scales", c_void_p),
                ("rotations", c_void_p)]


class GsAdapterOutGrads(Structure):
    _fields_ = [("means", c_void_p), ("covariances", c_void_p), ("harmonics", c_void_p), ("scales", c_void_p),
                ("rotations", c_void_p)]


class GsAdapterInGrads(Structure):
    _fields_ = [("coordinates", c_void_p), ("depths", c_void_p), ("raw_gaussians", c_void_p), ("c2w", c_void_p),
                ("kinv", c_void_p), ("multiplier", c_void_p)]


class GsLossConfig(Structure):
    _fields_ = [("batch", c_int32), ("channels", c_int32), ("height", c_int32), ("width", c_int32),
                ("pred_stride", c_int64), ("gt_stride", c_int64), ("with_mse", c_int32), ("reserved_", c_int32)]


class GsLpipsConfig(Structure):
    _fields_ = [("batch", c_int32), ("height", c_int32), ("width", c_int32), ("normalize", c_int32),
                ("in0_stride", c_int64), ("in1_stride", c_int64), ("grads", c_int32), ("reserved_", c_int32)]


SYMBOLS = {
    "gs_abi_version": (c_int, []),
    "gs_last_error": (c_char_p, []),
    "gs_context_create": (c_int, [POINTER(c_void_p)]),
    "gs_context_destroy": (None, [c_void_p]),
    "gs_context_trim": (c_int, [c_void_p]),
    "gs_forward": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), POINTER(GsOutputs), POINTER(c_void_p), c_void_p]),
    "gs_backward": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), c_void_p, POINTER(GsOutGrads),
                            POINTER(GsInGrads), c_void_p]),
    "gs_saved_free": (None, [c_void_p, c_void_p, c_void_p]),
    "gs_mark_visible": (c_int, [c_void_p, POINTER(GsConfig), c_void_p, c_void_p, c_void_p]),
    "gs_get_stats": (c_int, [c_void_p, POINTER(GsStats)]),
    "gs_render_host": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), POINTER(GsOutputs), c_void_p]),
    "gs_set_profiling": (c_int, [c_void_p, c_int]),
    "gs_get_stage_ms": (c_int, [c_void_p, POINTER(c_float)]),
    "gs_psnr_scratch_floats": (c_int64, [c_int32, c_int64]),
    "gs_psnr": (c_int, [c_void_p, c_void_p, c_int32, c_int64, c_void_p, c_void_p, c_void_p]),
    "gs_view_batch": (c_int, [c_int32, c_int32] + [c_void_p] * 10),
    "gs_ssim_scratch_floats": (c_int64, [c_int32, c_int32, c_int32, c_int32]),
    "gs_ssim": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "gs_adapter_forward": (c_int, [POINTER(GsAdapterConfig), POINTER(GsAdapterInputs), POINTER(GsAdapterOutputs), c_void_p]),
    "gs_adapter_backward": (c_int, [POINTER(GsAdapterConfig), POINTER(GsAdapterInputs), POINTER(GsAdapterOutGrads),
                                    POINTER(GsAdapterInGrads), c_void_p]),
    "gs_photometric_scratch_bytes": (c_int64, [POINTER(GsLossConfig)]),
    "gs_photometric_forward": (c_int, [POINTER(GsLossConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_photometric_backward": (c_int, [POINTER(GsLossConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p]),
    "gs_lpips_weights_create": (c_int, [POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_void_p,
                                        c_void_p, POINTER(c_void_p)]),
    "gs_lpips_weights_destroy": (None, [c_void_p]),
    "gs_lpips_workspace_bytes": (c_int64, [POINTER(GsLpipsConfig)]),
    "gs_lpips_forward": (c_int, [c_void_p, POINTER(GsLpipsConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_lpips_backward": (c_int, [c_void_p, POINTER(GsLpipsConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
}


class GsError(RuntimeError):
    pass


_lib = None


def lib() -> ctypes.CDLL:
    """Loads libgsplat_b200.so once; raises if it is absent (run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: the sm_90a extension has not been built "
                f"(sh pf3plat_b200/csrc/build.sh).  There is no CPU or PyTorch fallback.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the library does not export it
            fn.restype = res
            fn.argtypes = args
        if L.gs_abi_version() != ABI_VERSION:
            raise ImportError(f"{LIB_PATH}: ABI version {L.gs_abi_version()} != expected {ABI_VERSION}")
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().gs_last_error()
        text = msg.decode() if msg else "unknown error"
        if rc == -1:
            raise ValueError(text)  # same exception type the reference op raises for bad argument combinations
        raise GsError(f"gsplat_b200 error {rc}: {text}")
