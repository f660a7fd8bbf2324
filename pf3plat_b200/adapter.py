"""Fused Gaussian adapter: same class, config and `forward` signature as the reference's
PF3plat's src/model/encoder/common/gaussian_adapter.py:13-121, backed by the two CUDA kernels of
pf3plat_b200/csrc/gs_adapter.cu through the C ABI (gs_adapter_forward / gs_adapter_backward).

What changes for the caller: nothing but speed and memory.  `Gaussians.harmonics` has the reference's shape
(*batch, 3, d_sh) but is the transposed VIEW of a (*batch, d_sh, 3) buffer -- the layout the rasterizer reads -- so
the `rearrange(...).contiguous()` of PF3plat's src/model/decoder/cuda_splatting.py:75 becomes free.
There is no CPU / PyTorch fallback: without the CUDA library the import of pf3plat_b200._capi fails.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from math import prod

import torch
from torch import Tensor, nn

from . import _capi
from .sh_rotation import rotations_are_proper, sh_rotation_blocks


@dataclass
class Gaussians:  # gaussian_adapter.py:13-20
    means: Tensor
    covariances: Tensor
    scales: Tensor
    rotations: Tensor
    harmonics: Tensor
    opacities: Tensor


@dataclass
class GaussianAdapterCfg:  # gaussian_adapter.py:23-27
    gaussian_scale_min: float
    gaussian_scale_max: float
    sh_degree: int


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _f32c(t):
    return t.detach().to(torch.float32).contiguous()


class _AdapterFn(torch.autograd.Function):
    """inputs: c2w (V,4,4), kinv (V,3,3), multiplier (V,), sh_rotation (V,d,d)|None, sh_mask (d,), coordinates (V,R,2),
    depths (V,R), raw (V,R,7+3d).  outputs: means, covariances, harmonics (V,R,d,3), scales, rotations."""

    @staticmethod
    def forward(ctx, c2w, kinv, multiplier, sh_rotation, sh_mask, coordinates, depths, raw, scale_min, scale_max, eps):
        if not raw.is_cuda:
            raise RuntimeError("pf3plat_b200.adapter: tensors must live on a CUDA device (there is no CPU path)")
        V, R = depths.shape
        d_sh = sh_mask.shape[0]
        dev = raw.device
        keep = [_f32c(c2w), _f32c(kinv), _f32c(multiplier), None if sh_rotation is None else _f32c(sh_rotation),
                _f32c(sh_mask), _f32c(coordinates), _f32c(depths), _f32c(raw)]
        cfg = _capi.GsAdapterConfig(V=V, R=R, d_sh=d_sh, scale_min=scale_min, scale_max=scale_max, eps=eps,
                                    c2w=_ptr(keep[0]), kinv=_ptr(keep[1]), multiplier=_ptr(keep[2]),
                                    sh_rotation=_ptr(keep[3]), sh_mask=_ptr(keep[4]))
        inp = _capi.GsAdapterInputs(coordinates=_ptr(keep[5]), depths=_ptr(keep[6]), raw_gaussians=_ptr(keep[7]))
        means = torch.empty(V, R, 3, device=dev)
        cov = torch.empty(V, R, 3, 3, device=dev)
        harm = torch.empty(V, R, d_sh, 3, device=dev)
        scales = torch.empty(V, R, 3, device=dev)
        rot = torch.empty(V, R, 4, device=dev)
        out = _capi.GsAdapterOutputs(means=_ptr(means), covariances=_ptr(cov), harmonics=_ptr(harm), scales=_ptr(scales),
                                     rotations=_ptr(rot))
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _capi.check(_capi.lib().gs_adapter_forward(ctypes.byref(cfg), ctypes.byref(inp), ctypes.byref(out), stream))
        ctx.keep = keep
        ctx.consts = (V, R, d_sh, scale_min, scale_max, eps)
        return means, cov, harm, scales, rot

    @staticmethod
    def backward(ctx, g_means, g_cov, g_harm, g_scales, g_rot):
        V, R, d_sh, scale_min, scale_max, eps = ctx.consts
        keep = ctx.keep
        dev = keep[7].device
        need = ctx.needs_input_grad  # c2w, kinv, multiplier, sh_rotation, sh_mask, coordinates, depths, raw
        gs = [None if g is None else _f32c(g) for g in (g_means, g_cov, g_harm, g_scales, g_rot)]
        d_c2w = torch.empty(V, 4, 4, device=dev) if need[0] else None
        d_kinv = torch.empty(V, 3, 3, device=dev) if need[1] else None
        d_mult = torch.empty(V, device=dev) if need[2] else None
        d_coord = torch.empty(V, R, 2, device=dev) if need[5] else None
        d_depth = torch.empty(V, R, device=dev) if need[6] else None
        d_raw = torch.empty(V, R, 7 + 3 * d_sh, device=dev) if need[7] else None
        cfg = _capi.GsAdapterConfig(V=V, R=R, d_sh=d_sh, scale_min=scale_min, scale_max=scale_max, eps=eps,
                                    c2w=_ptr(keep[0]), kinv=_ptr(keep[1]), multiplier=_ptr(keep[2]),
                                    sh_rotation=_ptr(keep[3]), sh_mask=_ptr(keep[4]))
        scratch = None
        if torch.are_deterministic_algorithms_enabled():
            # per-camera sums added in a fixed order instead of with float atomics: bit-reproducible dL/dc2w, dL/dKinv,
            # dL/dmultiplier
            cfg.flags = _capi.GS_ADAPTER_DETERMINISTIC
            nbytes = _capi.lib().gs_adapter_scratch_bytes(ctypes.byref(cfg))
            if nbytes < 0:
                raise ValueError(f"invalid adapter configuration (V={V}, R={R}, d_sh={d_sh})")
            scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        inp = _capi.GsAdapterInputs(coordinates=_ptr(keep[5]), depths=_ptr(keep[6]), raw_gaussians=_ptr(keep[7]))
        gout = _capi.GsAdapterOutGrads(means=_ptr(gs[0]), covariances=_ptr(gs[1]), harmonics=_ptr(gs[2]),
                                       scales=_ptr(gs[3]), rotations=_ptr(gs[4]))
        gin = _capi.GsAdapterInGrads(coordinates=_ptr(d_coord), depths=_ptr(d_depth), raw_gaussians=_ptr(d_raw),
                                     c2w=_ptr(d_c2w), kinv=_ptr(d_kinv), multiplier=_ptr(d_mult), scratch=_ptr(scratch))
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _capi.check(_capi.lib().gs_adapter_backward(ctypes.byref(cfg), ctypes.byref(inp), ctypes.byref(gout),
                                                        ctypes.byref(gin), stream))
        return d_c2w, d_kinv, d_mult, None, None, d_coord, d_depth, d_raw, None, None, None


class GaussianAdapter(nn.Module):
    cfg: GaussianAdapterCfg

    def __init__(self, cfg: GaussianAdapterCfg):
        super().__init__()
        self.cfg = cfg
        # gaussian_adapter.py:37-46: large DC component, small view-dependent components at initialisation
        self.register_buffer("sh_mask", torch.ones((self.d_sh,), dtype=torch.float32), persistent=False)
        for degree in range(1, self.cfg.sh_degree + 1):
            self.sh_mask[degree ** 2:(degree + 1) ** 2] = 0.1 * 0.25 ** degree

    def forward(self, extrinsics: Tensor, intrinsics: Tensor, coordinates: Tensor, depths: Tensor, opacities: Tensor,
                raw_gaussians: Tensor, image_shape: tuple[int, int], eps: float = 1e-8,
                sh_rotation: Tensor | None = None) -> Gaussians:
        """Arguments as gaussian_adapter.py:48-58 (all broadcastable against each other over their batch dims).
        `sh_rotation` optionally supplies the per-camera block-diagonal Wigner-D matrices (batch dims of `extrinsics`
        + (d_sh, d_sh)); by default they are derived from extrinsics[..., :3, :3] as the reference's rotate_sh does."""
        device = extrinsics.device
        batch = torch.broadcast_shapes(extrinsics.shape[:-2], intrinsics.shape[:-2], coordinates.shape[:-1], depths.shape,
                                       opacities.shape, raw_gaussians.shape[:-1])
        nb = len(batch)
        # the leading dims over which the cameras vary; everything after them is "Gaussians of one camera"
        cam = torch.broadcast_shapes(extrinsics.shape[:-2], intrinsics.shape[:-2])
        cam = (1,) * (nb - len(cam)) + tuple(cam)
        k = max((i + 1 for i in range(nb) if cam[i] != 1), default=0)
        V, R = prod(batch[:k]), prod(batch[k:])
        first = (slice(None),) * k + (0,) * (nb - k)
        ext_v = extrinsics.broadcast_to(*batch, 4, 4)[first].reshape(V, 4, 4)
        intr_v = intrinsics.broadcast_to(*batch, 3, 3)[first].reshape(V, 3, 3)

        h, w = image_shape
        pixel_size = 1 / torch.tensor((w, h), dtype=torch.float32, device=device)
        kinv = intr_v.inverse()                                                  # projection.py:88-90
        multiplier = self.get_scale_multiplier(intr_v, pixel_size)               # gaussian_adapter.py:66
        c2w_rot = ext_v[..., :3, :3].detach()                                    # gaussian_adapter.py:81
        if sh_rotation is not None:
            d = sh_rotation.reshape(-1, self.d_sh, self.d_sh)
            if d.shape[0] not in (1, V):
                raise ValueError(f"sh_rotation holds {d.shape[0]} matrices for {V} cameras")
            d = d.expand(V, self.d_sh, self.d_sh)
        elif self.d_sh == 1 or not rotations_are_proper(c2w_rot):                # sh_rotation.py:21-22
            d = None
        else:
            d = sh_rotation_blocks(c2w_rot, self.d_sh)

        coords = coordinates.broadcast_to(*batch, 2).reshape(V, R, 2)
        dep = depths.broadcast_to(batch).reshape(V, R)
        raw = raw_gaussians.broadcast_to(*batch, raw_gaussians.shape[-1]).reshape(V, R, raw_gaussians.shape[-1])
        if raw.shape[-1] != self.d_in:
            raise ValueError(f"raw_gaussians has {raw.shape[-1]} channels, expected {self.d_in}")
        means, cov, harm, scales, rot = _AdapterFn.apply(ext_v, kinv, multiplier, d, self.sh_mask, coords, dep, raw,
                                                         float(self.cfg.gaussian_scale_min),
                                                         float(self.cfg.gaussian_scale_max), float(eps))
        return Gaussians(
            means=means.reshape(*batch, 3),
            covariances=cov.reshape(*batch, 3, 3),
            harmonics=harm.reshape(*batch, self.d_sh, 3).transpose(-1, -2),
            opacities=opacities,
            scales=scales.reshape(*batch, 3),
            rotations=rot.reshape(*batch, 4),
        )

    def get_scale_multiplier(self, intrinsics: Tensor, pixel_size: Tensor, multiplier: float = 0.1) -> Tensor:
        # gaussian_adapter.py:100-111
        xy_multipliers = multiplier * torch.einsum("...ij,j->...i", intrinsics[..., :2, :2].inverse(), pixel_size)
        return xy_multipliers.sum(dim=-1)

    @property
    def d_sh(self) -> int:
        return (self.cfg.sh_degree + 1) ** 2

    @property
    def d_in(self) -> int:
        return 7 + 3 * self.d_sh
