"""ctypes binding of the C ABI in include/gsplat_b200.h (pf3plat_b200/csrc/libgsplat_b200.so).

This is the only place the shared library is loaded.  There is NO fallback: if the library is missing or
was built for another ABI version the import fails loudly (the product path never routes through the CPU
oracle or any PyTorch re-implementation).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int8, c_int32, c_int64, c_uint32, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libgsplat_b200.so")
ABI_VERSION = 5

GS_FLAG_DEPTH = 1
GS_FLAG_PREFILTERED = 2
GS_FLAG_DETERMINISTIC = 4
GS_FLAG_ANTIALIAS = 8
GS_DEPTH_Z = 0
GS_DEPTH_DISPARITY = 1
GS_DEPTH_RELATIVE_DISPARITY = 2
GS_DEPTH_LOG = 3
# PF3plat's DepthRenderingMode names -> GsConfig.depth_mode
DEPTH_MODES = {"depth": GS_DEPTH_Z, "disparity": GS_DEPTH_DISPARITY, "relative_disparity": GS_DEPTH_RELATIVE_DISPARITY,
               "log": GS_DEPTH_LOG}
GS_ADAPTER_DETERMINISTIC = 1
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
GS_TUNE_ALL_STRATA = 524288
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
        ("tanfov", c_void_p), ("view_scale", c_void_p), ("depth_mode", c_int32), ("depth_near_far", c_void_p),
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
                ("dL_dcov3D", c_void_p), ("dL_dviewmatrix_z", c_void_p)]


class GsAlpha(Structure):
    """The accumulated-opacity output of gs_forward_ex / gs_render_host_ex and its incoming gradient of gs_backward_ex."""
    _fields_ = [("alpha", c_void_p), ("dL_dalpha", c_void_p)]


class GsCameraGrads(Structure):
    """The camera gradient gs_backward_cam writes: dL/dviewmatrix [V,16], dL/dprojmatrix [V,16], dL/dcampos [V,3]."""
    _fields_ = [("dL_dviewmatrix", c_void_p), ("dL_dprojmatrix", c_void_p), ("dL_dcampos", c_void_p)]


class GsStats(Structure):
    _fields_ = [("num_rendered", c_int64), ("num_visible", c_int64), ("saved_bytes", c_int64),
                ("scratch_bytes", c_int64), ("kernel_launches", c_int32), ("max_tile_list", c_int32),
                ("speculative", c_int32), ("overflow_redos", c_int32), ("pool_reserved_bytes", c_int64),
                ("pool_used_bytes", c_int64)]


GS_SYNC_FREE_DETERMINISTIC = 1
GS_SYNC_FREE_CAMERA_GRAD = 2


class GsSyncFreeWorkspace(Structure):
    """A caller-owned workspace of gs_forward_sync_free / gs_backward_sync_free."""
    _fields_ = [("base", c_void_p), ("bytes", c_int64), ("instance_capacity", c_int64)]


# every symbol include/gsplat_b200.h declares: name -> (restype, argtypes)
class GsAdapterConfig(Structure):
    _fields_ = [("V", c_int32), ("R", c_int32), ("d_sh", c_int32), ("flags", c_uint32),
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
                ("kinv", c_void_p), ("multiplier", c_void_p), ("scratch", c_void_p)]


class GsLossConfig(Structure):
    _fields_ = [("batch", c_int32), ("channels", c_int32), ("height", c_int32), ("width", c_int32),
                ("pred_stride", c_int64), ("gt_stride", c_int64), ("with_mse", c_int32), ("reserved_", c_int32)]


GS_LPIPS_TF32, GS_LPIPS_BF16 = 0, 1
LPIPS_PRECISIONS = {"tf32": GS_LPIPS_TF32, "bf16": GS_LPIPS_BF16}


class GsLpipsConfig(Structure):
    _fields_ = [("batch", c_int32), ("height", c_int32), ("width", c_int32), ("normalize", c_int32),
                ("in0_stride", c_int64), ("in1_stride", c_int64), ("grads", c_int32), ("precision", c_int32)]


GsLpipsConfig.reserved_ = GsLpipsConfig.precision  # the header's other name for the field (a union member)


class GsPoseLossConfig(Structure):
    _fields_ = [("batch", c_int32), ("views", c_int32), ("height", c_int32), ("width", c_int32),
                ("segments", c_int32), ("reserved_", c_int32), ("matches", c_int64)]


class GsPoseLossInputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("T", "kinv_a", "k_c", "conf", "seg", "offsets", "id_a", "id_c", "w", "depth",
                                        "xyz")]


class GsPoseLossGrads(Structure):
    _fields_ = [(n, c_void_p) for n in ("dL_dT", "dL_ddepth", "dL_dxyz", "dL_dw", "dL_dconf")]


GS_COSTVOLUME_DETERMINISTIC = 1


class GsCostVolumeConfig(Structure):
    _fields_ = [("batch", c_int32), ("views", c_int32), ("channels", c_int32), ("height", c_int32), ("width", c_int32),
                ("depth_candidates", c_int32), ("intrinsics_rows", c_int32), ("flags", c_uint32),
                ("feat_stride", c_int64 * 5)]


class GsCostVolumeInputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("features", "intrinsics", "extrinsics", "near_", "far_")]


class GsCostVolumeGrads(Structure):
    _fields_ = [("dL_dcost", c_void_p), ("dL_dfeatures", c_void_p)]


GS_POSES_MAX_VIEWS = 16
GS_POSES_MAX_PAIRS = 120


class GsPoseSyncConfig(Structure):
    _fields_ = [("batch", c_int32), ("views", c_int32), ("pairs", c_int32), ("reserved_", c_int32),
                ("pair_i", c_int8 * GS_POSES_MAX_PAIRS), ("pair_j", c_int8 * GS_POSES_MAX_PAIRS)]


class GsRefinePosesConfig(Structure):
    _fields_ = [("batch", c_int32), ("views", c_int32)]


class GsRefinePosesInputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("pose_enc", "delta", "gamma")]


class GsRefinePosesGrads(Structure):
    _fields_ = [(n, c_void_p) for n in ("dL_dabspose", "dL_dabspose_inv", "dL_dpose_enc", "dL_ddelta", "dL_dgamma")]


class GsPluckerConfig(Structure):
    _fields_ = [("batch", c_int32), ("views", c_int32), ("height", c_int32), ("width", c_int32)]


class GsDepthUpdateConfig(Structure):
    _fields_ = [(n, c_int32) for n in ("batch", "views", "height", "width", "grid_height", "grid_width")]


class GsDepthUpdateInputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("depth", "scale_shift", "intrinsics", "near_", "far_")]


class GsDepthUpdateGrads(Structure):
    _fields_ = [(n, c_void_p) for n in ("dL_ddepths", "dL_dxyz", "dL_dscale_shift")]


GS_MONO_CUE_BINS = 128


class GsMonoCueConfig(Structure):
    _fields_ = [(n, c_int32) for n in ("batch", "views", "height", "width")]


class GsPdfPeakConfig(Structure):
    _fields_ = [(n, c_int32) for n in ("items", "depth_candidates", "height", "width", "upscale")]



class GsGaussianHeadConfig(Structure):
    _fields_ = [(n, c_int32) for n in ("batch", "views", "height", "width", "d_sh")] + [
        ("flags", c_uint32), ("scale_min", c_float), ("scale_max", c_float), ("eps", c_float), ("reserved_", c_int32)]


class GsGaussianHeadInputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("raw_gaussians", "density_logits", "depths", "c2w", "intrinsics", "sh_rotation",
                                        "sh_mask")]


class GsGaussianHeadOutputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("means", "covariances", "harmonics", "opacities")]


class GsGaussianHeadOutGrads(Structure):
    _fields_ = [(n, c_void_p) for n in ("means", "covariances", "harmonics", "opacities")]


class GsGaussianHeadInGrads(Structure):
    _fields_ = [(n, c_void_p) for n in ("raw_gaussians", "density_logits", "depths", "c2w", "scratch")]


class GsShRotationConfig(Structure):
    _fields_ = [("outer", c_int32), ("inner", c_int32), ("outer_stride", c_int64), ("inner_stride", c_int64),
                ("row_stride", c_int32), ("d_sh", c_int32)]


GS_ADAM_CHUNK = 16384


class GsAdamChunk(Structure):
    _fields_ = [(n, c_void_p) for n in ("param", "grad", "exp_avg", "exp_avg_sq")] + [
        ("begin", c_int64), ("count", c_int32), ("tensor", c_int32)]


class GsAdamConfig(Structure):
    _fields_ = [("tensors", c_int32), ("chunks", c_int32), ("beta1", c_double), ("beta2", c_double), ("eps", c_double),
                ("max_norm", c_double), ("zero_grads", c_int32), ("reserved_", c_int32)]


SYMBOLS = {
    "gs_abi_version": (c_int, []),
    "gs_last_error": (c_char_p, []),
    "gs_supported_flags": (c_uint32, []),
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
    "gs_forward_ex": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), POINTER(GsOutputs), POINTER(GsAlpha),
                              POINTER(c_void_p), c_void_p]),
    "gs_backward_ex": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), c_void_p, POINTER(GsOutGrads),
                               POINTER(GsAlpha), POINTER(GsInGrads), c_void_p]),
    "gs_backward_cam": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), c_void_p, POINTER(GsOutGrads),
                                POINTER(GsAlpha), POINTER(GsInGrads), POINTER(GsCameraGrads), c_void_p]),
    "gs_backward_cam_tanfov": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), c_void_p, POINTER(GsOutGrads),
                                       POINTER(GsAlpha), POINTER(GsInGrads), POINTER(GsCameraGrads), c_void_p,
                                       c_void_p]),
    "gs_render_host_ex": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), POINTER(GsOutputs), POINTER(GsAlpha),
                                  c_void_p]),
    "gs_sync_free_workspace_bytes": (c_int, [POINTER(GsConfig), c_int64, c_uint32, POINTER(c_int64)]),
    "gs_forward_sync_free": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), POINTER(GsOutputs), POINTER(GsAlpha),
                                     POINTER(GsSyncFreeWorkspace), POINTER(c_void_p), c_void_p]),
    "gs_backward_sync_free": (c_int, [c_void_p, POINTER(GsConfig), POINTER(GsInputs), c_void_p, POINTER(GsOutGrads),
                                      POINTER(GsAlpha), POINTER(GsInGrads), POINTER(GsCameraGrads), c_void_p,
                                      POINTER(GsSyncFreeWorkspace), c_void_p]),
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
    "gs_adapter_scratch_bytes": (c_int64, [POINTER(GsAdapterConfig)]),
    "gs_photometric_scratch_bytes": (c_int64, [POINTER(GsLossConfig)]),
    "gs_photometric_forward": (c_int, [POINTER(GsLossConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_photometric_backward": (c_int, [POINTER(GsLossConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p]),
    "gs_lpips_weights_create": (c_int, [POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_void_p,
                                        c_void_p, POINTER(c_void_p)]),
    "gs_lpips_weights_pack_bf16": (c_int, [c_void_p, POINTER(c_void_p), c_void_p]),
    "gs_lpips_weights_destroy": (None, [c_void_p]),
    "gs_lpips_workspace_bytes": (c_int64, [POINTER(GsLpipsConfig)]),
    "gs_lpips_forward": (c_int, [c_void_p, POINTER(GsLpipsConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_lpips_backward": (c_int, [c_void_p, POINTER(GsLpipsConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_pose_loss_scratch_bytes": (c_int64, [POINTER(GsPoseLossConfig)]),
    "gs_pose_loss_forward": (c_int, [POINTER(GsPoseLossConfig), POINTER(GsPoseLossInputs), c_void_p, c_void_p, c_void_p]),
    "gs_pose_loss_backward": (c_int, [POINTER(GsPoseLossConfig), POINTER(GsPoseLossInputs), c_void_p, c_void_p,
                                      POINTER(GsPoseLossGrads), c_void_p, c_void_p]),
    "gs_costvolume_scratch_bytes": (c_int64, [POINTER(GsCostVolumeConfig), c_int32]),
    "gs_costvolume_forward": (c_int, [POINTER(GsCostVolumeConfig), POINTER(GsCostVolumeInputs), c_void_p, c_void_p,
                                      c_void_p]),
    "gs_costvolume_backward": (c_int, [POINTER(GsCostVolumeConfig), POINTER(GsCostVolumeInputs),
                                       POINTER(GsCostVolumeGrads), c_void_p, c_void_p]),
    "gs_pose_sync_scratch_bytes": (c_int64, [POINTER(GsPoseSyncConfig)]),
    "gs_pose_sync": (c_int, [POINTER(GsPoseSyncConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_refine_poses_forward": (c_int, [POINTER(GsRefinePosesConfig), POINTER(GsRefinePosesInputs), c_void_p, c_void_p,
                                        c_void_p]),
    "gs_refine_poses_backward": (c_int, [POINTER(GsRefinePosesConfig), POINTER(GsRefinePosesInputs),
                                         POINTER(GsRefinePosesGrads), c_void_p]),
    "gs_plucker_rays": (c_int, [POINTER(GsPluckerConfig), c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_depth_update_forward": (c_int, [POINTER(GsDepthUpdateConfig), POINTER(GsDepthUpdateInputs), c_void_p, c_void_p,
                                        c_void_p]),
    "gs_depth_update_backward": (c_int, [POINTER(GsDepthUpdateConfig), POINTER(GsDepthUpdateInputs),
                                         POINTER(GsDepthUpdateGrads), c_void_p]),
    "gs_mono_cue": (c_int, [POINTER(GsMonoCueConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_pdf_peak_forward": (c_int, [POINTER(GsPdfPeakConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_pdf_peak_backward": (c_int, [POINTER(GsPdfPeakConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p]),
    "gs_gaussian_head_scratch_bytes": (c_int64, [POINTER(GsGaussianHeadConfig)]),
    "gs_gaussian_head_forward": (c_int, [POINTER(GsGaussianHeadConfig), POINTER(GsGaussianHeadInputs),
                                         POINTER(GsGaussianHeadOutputs), c_void_p]),
    "gs_gaussian_head_backward": (c_int, [POINTER(GsGaussianHeadConfig), POINTER(GsGaussianHeadInputs),
                                          POINTER(GsGaussianHeadOutGrads), POINTER(GsGaussianHeadInGrads), c_void_p]),
    "gs_sh_rotation_workspace_bytes": (c_int64, [POINTER(GsShRotationConfig)]),
    "gs_sh_rotation_blocks": (c_int, [POINTER(GsShRotationConfig), c_void_p, c_void_p, c_void_p, c_void_p]),
    "gs_adam_scratch_bytes": (c_int64, [POINTER(GsAdamConfig)]),
    "gs_adam_step": (c_int, [POINTER(GsAdamConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
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
