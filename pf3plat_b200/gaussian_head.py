"""PF3plat's Gaussian head on the device (csrc/gs_gaussian_head.cu): from the depth predictor's two output convolutions to
the Gaussians the encoder returns, in one call, forward and backward.

`gaussian_head(raw_gaussians, density_logits, depths, c2w, intrinsics, adapter_cfg, image_shape)` replaces
depth_predictor_multiview.py:397-415 (the rearrange of to_gaussians' output, the sigmoid of to_disparity's density
channel and its repeat), encoder_costvolume.py:509-540 (the pixel grid and its learned offset, the opacity map, the
[:, (0, -1)] selections and the adapter call) and :556-573 (the b (v r srf spp) rearrange of every output), for
gaussians_per_pixel = num_surfaces = 1.  Views 0 and V - 1 are selected inside the kernel; nothing is gathered.

Nothing here synchronises the device with the host: K^-1 and the scale multiplier are computed per camera on the device,
and the reference's SH rotation guard (sh_rotation.py:21, every determinant allclose to 1 or every camera uses the
identity) is a device flag that the Wigner-D kernel reads (csrc/gs_sh_rotation.cu).  The backward reduces the per-camera dL/dc2w in a fixed order without
atomics, so it is bit-reproducible with or without torch.use_deterministic_algorithms.  Inputs must be float32 CUDA
tensors; there is no CPU fallback.

Scales and rotations are not produced: only visualization_dump reads them, and a run that dumps keeps the adapter call
for the dump.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import torch
from torch import Tensor

from . import _capi
from .adapter import GaussianAdapterCfg
from .sh_rotation import guarded_sh_rotation_blocks

_MASKS: dict = {}


@dataclass
class HeadGaussians:
    """The four fields of PF3plat's model/types.py Gaussians, G = 2 h w per scene.  `harmonics` [b, G, 3, d_sh] is the
    transposed view of a [b, G, d_sh, 3] buffer, the layout the rasterizer reads."""
    means: Tensor
    covariances: Tensor
    harmonics: Tensor
    opacities: Tensor


def _check(name, t, dev=None):
    if not torch.is_tensor(t):
        raise TypeError(f"gaussian_head: {name} must be a tensor")
    if t.device.type != "cuda":
        raise TypeError(f"gaussian_head: {name} must be a CUDA tensor (there is no CPU fallback), got {t.device}")
    if t.dtype != torch.float32:
        raise TypeError(f"gaussian_head: {name} must be float32, got {t.dtype}")
    if dev is not None and t.device != dev:
        raise ValueError(f"gaussian_head: {name} is on {t.device}, expected {dev}")


def _sh_mask(sh_degree, dev):
    """gaussian_adapter.py:39-46, built on the device once per (degree, device)"""
    key = (sh_degree, dev)
    if key not in _MASKS:
        m = torch.ones(((sh_degree + 1) ** 2,), dtype=torch.float32, device=dev)
        for degree in range(1, sh_degree + 1):
            m[degree ** 2:(degree + 1) ** 2] = 0.1 * 0.25 ** degree
        _MASKS[key] = m
    return _MASKS[key]


def sh_rotation_for_slots(c2w: Tensor, d_sh: int) -> Tensor | None:
    """[b, 2, d_sh, d_sh] block-diagonal Wigner-D matrices of c2w[:, (0, -1), :3, :3].detach() after the reference's
    all-or-nothing guard (sh_rotation.py:21-22: unless every determinant is allclose to 1, every camera of the call uses
    the identity; a NaN determinant fails), built on the device in two launches (csrc/gs_sh_rotation.cu) from the
    strided view of views 0 and V - 1.  None for d_sh = 1."""
    if d_sh == 1:
        return None
    return guarded_sh_rotation_blocks(c2w.detach()[:, ::c2w.shape[1] - 1], d_sh)


def _structs(raw, logits, depths, c2w, intrinsics, sh_rot, sh_mask, consts):
    b, V, h, w, d_sh, smin, smax, eps = consts
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    cfg = _capi.GsGaussianHeadConfig(batch=b, views=V, height=h, width=w, d_sh=d_sh, scale_min=smin, scale_max=smax,
                                     eps=eps)
    ins = _capi.GsGaussianHeadInputs(raw_gaussians=ptr(raw), density_logits=ptr(logits), depths=ptr(depths),
                                     c2w=ptr(c2w), intrinsics=ptr(intrinsics), sh_rotation=ptr(sh_rot),
                                     sh_mask=ptr(sh_mask))
    return cfg, ins


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


class _GaussianHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw, logits, depths, c2w, intrinsics, sh_rot, sh_mask, consts):
        b, V, h, w, d_sh = consts[:5]
        G, dev = 2 * h * w, raw.device
        cfg, ins = _structs(raw, logits, depths, c2w, intrinsics, sh_rot, sh_mask, consts)
        means = torch.empty(b, G, 3, device=dev)
        cov = torch.empty(b, G, 3, 3, device=dev)
        harm = torch.empty(b, G, d_sh, 3, device=dev)
        opac = torch.empty(b, G, device=dev)
        out = _capi.GsGaussianHeadOutputs(means=means.data_ptr(), covariances=cov.data_ptr(),
                                          harmonics=harm.data_ptr(), opacities=opac.data_ptr())
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_gaussian_head_forward(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(out),
                                                             _stream(dev)))
        ctx.save_for_backward(raw, logits, depths, c2w, intrinsics, sh_rot, sh_mask)
        ctx.consts = consts
        ctx.set_materialize_grads(False)
        return means, cov, harm, opac

    @staticmethod
    def backward(ctx, g_means, g_cov, g_harm, g_opac):
        none = (None,) * 8
        if g_means is None and g_cov is None and g_harm is None and g_opac is None:
            return none
        raw, logits, depths, c2w, intrinsics, sh_rot, sh_mask = ctx.saved_tensors
        consts = ctx.consts
        dev = raw.device
        need = ctx.needs_input_grad
        gs = [None if g is None else g.to(torch.float32).contiguous() for g in (g_means, g_cov, g_harm, g_opac)]
        d_raw = torch.empty_like(raw) if need[0] else None
        d_logits = torch.empty_like(logits) if need[1] else None
        d_depths = torch.empty_like(depths) if need[2] else None
        d_c2w = torch.empty_like(c2w) if need[3] else None
        cfg, ins = _structs(raw, logits, depths, c2w, intrinsics, sh_rot, sh_mask, consts)
        scratch = None
        if d_c2w is not None:
            nbytes = _capi.lib().gs_gaussian_head_scratch_bytes(ctypes.byref(cfg))
            if nbytes < 0:
                raise ValueError(f"gaussian_head: invalid configuration {consts}")
            scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        gout = _capi.GsGaussianHeadOutGrads(means=ptr(gs[0]), covariances=ptr(gs[1]), harmonics=ptr(gs[2]),
                                            opacities=ptr(gs[3]))
        gin = _capi.GsGaussianHeadInGrads(raw_gaussians=ptr(d_raw), density_logits=ptr(d_logits),
                                          depths=ptr(d_depths), c2w=ptr(d_c2w), scratch=ptr(scratch))
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_gaussian_head_backward(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(gout),
                                                              ctypes.byref(gin), _stream(dev)))
        return d_raw, d_logits, d_depths, d_c2w, None, None, None, None


def gaussian_head(raw_gaussians: Tensor, density_logits: Tensor, depths: Tensor, c2w: Tensor, intrinsics: Tensor,
                  adapter_cfg: GaussianAdapterCfg, image_shape, eps: float = 1e-8, gaussians_per_pixel: int = 1,
                  num_surfaces: int = 1) -> HeadGaussians:
    """raw_gaussians: to_gaussians' output [(v b), 9 + 3 d_sh, h, w] with v = 2 depth-predictor views;
    density_logits: to_disparity's output [(v b), 2, h, w] (channel 1 the raw density, channel 0 unused);
    depths: depth_update's depths [(b V), 1, h, w] over all V >= 2 context views; c2w: refine_poses' second output
    [b, V, 4, 4]; intrinsics: the context's normalised [b, V, 3, 3] (data: must not require grad);
    image_shape: (h, w).  Returns the encoder's Gaussians of views 0 and V - 1, G = 2 h w per scene.  Gradients reach
    raw_gaussians, density_logits, depths and c2w (through the means only)."""
    _check("raw_gaussians", raw_gaussians)
    dev = raw_gaussians.device
    for name, t in (("density_logits", density_logits), ("depths", depths), ("c2w", c2w), ("intrinsics", intrinsics)):
        _check(name, t, dev)
    if gaussians_per_pixel != 1 or num_surfaces != 1:
        raise ValueError(f"gaussian_head supports gaussians_per_pixel = num_surfaces = 1 (every PF3plat config), got "
                         f"{gaussians_per_pixel}, {num_surfaces}")
    deg = adapter_cfg.sh_degree
    if not isinstance(deg, int) or not 0 <= deg <= 4:
        raise ValueError(f"gaussian_head: sh_degree must be an integer in [0, 4] (d_sh a square <= 25), got {deg!r}")
    d_sh = (deg + 1) ** 2
    h, w = (int(x) for x in image_shape)
    if c2w.dim() != 4 or c2w.shape[2:] != (4, 4) or c2w.shape[0] < 1 or c2w.shape[1] < 2:
        raise ValueError(f"gaussian_head needs c2w [b, V, 4, 4] with V >= 2, got {tuple(c2w.shape)}")
    b, V = c2w.shape[:2]
    if tuple(intrinsics.shape) != (b, V, 3, 3):
        raise ValueError(f"gaussian_head needs intrinsics [b, V, 3, 3] = [{b}, {V}, 3, 3], got {tuple(intrinsics.shape)}")
    if h < 1 or w < 1 or tuple(depths.shape) != (b * V, 1, h, w):
        raise ValueError(f"gaussian_head needs depths [(b V), 1, h, w] = [{b * V}, 1, {h}, {w}], got "
                         f"{tuple(depths.shape)}")
    C = 9 + 3 * d_sh
    if raw_gaussians.dim() != 4 or raw_gaussians.shape[1] != C:
        raise ValueError(f"gaussian_head needs raw_gaussians with 2 + 7 + 3 d_sh = {C} channels (sh_degree {deg}), got "
                         f"{tuple(raw_gaussians.shape)}")
    if tuple(raw_gaussians.shape) != (2 * b, C, h, w):
        raise ValueError(f"gaussian_head needs raw_gaussians [(v b), {C}, h, w] with v = 2 depth-predictor views and "
                         f"b = {b}: [{2 * b}, {C}, {h}, {w}], got {tuple(raw_gaussians.shape)}")
    if tuple(density_logits.shape) != (2 * b, 2, h, w):
        raise ValueError(f"gaussian_head needs density_logits [(v b), 2, h, w] = [{2 * b}, 2, {h}, {w}], got "
                         f"{tuple(density_logits.shape)}")
    if intrinsics.requires_grad:
        raise ValueError("gaussian_head: intrinsics must not require grad (they are data in PF3plat)")
    with torch.cuda.device(dev):
        sh_rot = sh_rotation_for_slots(c2w, d_sh)
        consts = (b, V, h, w, d_sh, float(adapter_cfg.gaussian_scale_min), float(adapter_cfg.gaussian_scale_max),
                  float(eps))
        means, cov, harm, opac = _GaussianHead.apply(raw_gaussians.contiguous(), density_logits.contiguous(),
                                                     depths.contiguous(), c2w.contiguous(), intrinsics.contiguous(),
                                                     sh_rot, _sh_mask(deg, dev), consts)
    return HeadGaussians(means=means, covariances=cov, harmonics=harm.transpose(-1, -2), opacities=opac)
