"""PF3plat's plane-sweep cost volume on the device (csrc/gs_costvolume.cu).

`plane_sweep_cost_volume` is the parameter-free part of `DepthPredictorMultiView.forward`
(src/model/encoder/costvolume/depth_predictor_multiview.py:309-343): for every depth candidate, warp the other views'
features into each view and correlate them with its own, averaged over the other views.  It returns
`raw_correlation_in` before the `torch.cat` with `feat01`, [(v b), D, h, w] in the reference's (v b) order, without ever
storing the [(v b), C, D, h, w] warped feature volume.

Gradients reach `features` only, in both of its roles (the target features and the sampled source features).  As in
the reference, the sampling grid is built under no_grad and the intrinsics, near and far are detached, so the
cameras get no gradient from this op even when they require grad.  Under `torch.use_deterministic_algorithms(True)`
the backward is bit-reproducible (exact fixed-point accumulation of the source role); otherwise it adds float atomics.
Inputs must be float32 CUDA tensors; there is no CPU fallback.
"""
from __future__ import annotations

import torch

from . import _capi


def _config(features, rows: int, D: int, deterministic: bool) -> _capi.GsCostVolumeConfig:
    b, v, C, h, w = features.shape
    cfg = _capi.GsCostVolumeConfig(batch=b, views=v, channels=C, height=h, width=w, depth_candidates=D,
                                   intrinsics_rows=rows,
                                   flags=_capi.GS_COSTVOLUME_DETERMINISTIC if deterministic else 0)
    for i, s in enumerate(features.stride()):
        cfg.feat_stride[i] = s
    return cfg


def _inputs(features, K, E, near, far) -> _capi.GsCostVolumeInputs:
    return _capi.GsCostVolumeInputs(features=features.data_ptr(), intrinsics=K.data_ptr(), extrinsics=E.data_ptr(),
                                    near_=near.data_ptr(), far_=far.data_ptr())


def _scratch(L, cfg, backward: bool, dev):
    nbytes = int(L.gs_costvolume_scratch_bytes(cfg, 1 if backward else 0))
    if nbytes < 0:
        _capi.check(-1)
    return torch.empty((nbytes,), dtype=torch.uint8, device=dev)


class _CostVolume(torch.autograd.Function):
    """features [b, v, C, h, w] (any strides); cameras as constants -> cost [(v b), D, h, w]."""

    @staticmethod
    def forward(ctx, features, K, E, near, far, D):
        b, v, _, h, w = features.shape
        dev = features.device
        cfg = _config(features, K.shape[-1], D, False)
        out = torch.empty((v * b, D, h, w), dtype=torch.float32, device=dev)
        L = _capi.lib()
        with torch.cuda.device(dev):
            scratch = _scratch(L, cfg, False, dev)
            _capi.check(L.gs_costvolume_forward(cfg, _inputs(features, K, E, near, far), out.data_ptr(),
                                                scratch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(features, K, E, near, far)
        ctx.D = D
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, dcost):
        if dcost is None or not ctx.needs_input_grad[0]:
            return (None,) * 6
        features, K, E, near, far = ctx.saved_tensors
        dev = features.device
        cfg = _config(features, K.shape[-1], ctx.D, torch.are_deterministic_algorithms_enabled())
        g = dcost.to(torch.float32).contiguous()
        dfeat = torch.empty(features.shape, dtype=torch.float32, device=dev)
        grads = _capi.GsCostVolumeGrads(dL_dcost=g.data_ptr(), dL_dfeatures=dfeat.data_ptr())
        L = _capi.lib()
        with torch.cuda.device(dev):
            scratch = _scratch(L, cfg, True, dev)
            _capi.check(L.gs_costvolume_backward(cfg, _inputs(features, K, E, near, far), grads, scratch.data_ptr(),
                                                 torch.cuda.current_stream(dev).cuda_stream))
        return dfeat, None, None, None, None, None


def plane_sweep_cost_volume(features: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                            near: torch.Tensor, far: torch.Tensor, num_depth_candidates: int) -> torch.Tensor:
    """`raw_correlation_in` of DepthPredictorMultiView.forward (depth_predictor_multiview.py:341-343, before the
    torch.cat): [(v b), D, h, w].

    features [b, v, C, h, w] (any strides); intrinsics [b, v, 3, 3] or [b, v, 4, 4] (normalised, read through
    [..., :3, :3]); extrinsics [b, v, 4, 4] camera-to-world; near, far [b, v].  Needs v >= 2 and h, w >= 2.
    Differentiable with respect to `features` only."""
    tensors = {"features": features, "intrinsics": intrinsics, "extrinsics": extrinsics, "near": near, "far": far}
    for name, t in tensors.items():
        if not torch.is_tensor(t) or t.device.type != "cuda":
            raise RuntimeError(f"plane_sweep_cost_volume needs {name} as a CUDA tensor (there is no CPU fallback)")
        if t.dtype != torch.float32:
            raise TypeError(f"plane_sweep_cost_volume needs float32 {name}, got {t.dtype}")
        if t.device != features.device:
            raise ValueError(f"plane_sweep_cost_volume: {name} is on {t.device}, features on {features.device}")
    if features.dim() != 5:
        raise ValueError(f"plane_sweep_cost_volume: features must be [b, v, C, h, w], got {tuple(features.shape)}")
    b, v, C, h, w = features.shape
    D = int(num_depth_candidates)
    rows = intrinsics.shape[-1] if intrinsics.dim() == 4 else 0
    if (tuple(intrinsics.shape) != (b, v, rows, rows) or rows not in (3, 4) or tuple(extrinsics.shape) != (b, v, 4, 4)
            or tuple(near.shape) != (b, v) or tuple(far.shape) != (b, v)):
        raise ValueError(f"plane_sweep_cost_volume: shapes disagree with features {tuple(features.shape)}: intrinsics "
                         f"{tuple(intrinsics.shape)}, extrinsics {tuple(extrinsics.shape)}, near {tuple(near.shape)}, "
                         f"far {tuple(far.shape)}")
    if b < 1 or v < 2 or C < 1 or h < 2 or w < 2 or D < 1:
        raise ValueError(f"plane_sweep_cost_volume needs b >= 1, v >= 2, C >= 1, h >= 2, w >= 2 and at least one depth "
                         f"candidate; got features {tuple(features.shape)}, num_depth_candidates={D}")
    cams = [t.detach().contiguous() for t in (intrinsics, extrinsics, near, far)]
    return _CostVolume.apply(features, *cams, D)
