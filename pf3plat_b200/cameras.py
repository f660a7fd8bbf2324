"""Camera glue of the render boundary, batched over views.

Restates what `render_cuda` does before its per-view loop
(PF3plat's src/model/decoder/cuda_splatting.py:64-87) so that the batched
entry (`pf3plat_b200.render`) can be fed the same arguments as the reference
function.  On CUDA tensors `make_view_batch` is ONE kernel (gs_view_batch,
csrc/gs_cameras.cu) instead of ~50 small tensor ops with two cuSOLVER inversions;
on CPU tensors (how the tests prepare the oracle's inputs) it is the same
arithmetic in plain tensor code.  The drop-in `GaussianRasterizer` does not need
this module: there the reference's own glue runs unmodified and hands us finished
matrices.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch


def get_fov(intrinsics: torch.Tensor) -> torch.Tensor:
    """(B,3,3) normalised intrinsics -> (B,2) full fov (x,y) in radians
    (PF3plat's src/geometry/projection.py:233-247)."""
    inv = torch.linalg.inv(intrinsics)

    def ray(v):
        v = torch.tensor(v, dtype=intrinsics.dtype, device=intrinsics.device)
        d = torch.einsum("bij,j->bi", inv, v)
        return d / d.norm(dim=-1, keepdim=True)

    fov_x = (ray([0.0, 0.5, 1.0]) * ray([1.0, 0.5, 1.0])).sum(-1).acos()
    fov_y = (ray([0.5, 0.0, 1.0]) * ray([0.5, 1.0, 1.0])).sum(-1).acos()
    return torch.stack((fov_x, fov_y), dim=-1)


def get_projection_matrix(near, far, fov_x, fov_y) -> torch.Tensor:
    """z in [0,1] perspective matrix, principal point centred
    (PF3plat's src/model/decoder/cuda_splatting.py:17-44)."""
    tx, ty = (0.5 * fov_x).tan(), (0.5 * fov_y).tan()
    top, right = ty * near, tx * near
    bottom, left = -top, -right
    (b,) = near.shape
    m = torch.zeros((b, 4, 4), dtype=near.dtype, device=near.device)
    m[:, 0, 0] = 2 * near / (right - left)
    m[:, 1, 1] = 2 * near / (top - bottom)
    m[:, 0, 2] = (right + left) / (right - left)
    m[:, 1, 2] = (top + bottom) / (top - bottom)
    m[:, 3, 2] = 1
    m[:, 2, 2] = far / (far - near)
    m[:, 2, 3] = -(far * near) / (far - near)
    return m


@dataclass
class ViewBatch:
    """Per-view camera block in the layout the C-ABI takes (include/gsplat_b200.h: GsView arrays)."""
    viewmatrix: torch.Tensor   # (V,4,4) transposed world->camera
    projmatrix: torch.Tensor   # (V,4,4) transposed full projection
    campos: torch.Tensor       # (V,3)
    tanfov: torch.Tensor       # (V,2)
    scale: torch.Tensor        # (V,) the 1/near rescale applied to means/covariances (1 if not scale-invariant)


def make_view_batch(extrinsics, intrinsics, near, far, scale_invariant: bool = True,
                    camera_gradients=None) -> ViewBatch:
    """cuda_splatting.py:64-87 for all views at once (no per-view `.item()` host syncs).

    On CUDA tensors whose extrinsics require grad, `viewmatrix` is differentiable w.r.t. them: its values are the
    kernel's, its gradient that of the view matrix built in torch.  This is what lets the fused depth channel carry
    render_depth_cuda's camera gradient (cuda_splatting.py:239-242).  `projmatrix`, `campos` and `tanfov` stay
    detached, and `near` / `far` get no gradient.

    camera_gradients (None = rasterizer.get_camera_gradients()): on, with extrinsics or intrinsics that require grad, the
    camera inputs follow render_cuda's own torch glue instead -- the translation of the extrinsics rescaled by 1/near,
    then inverted; projmatrix = view @ P, P from the fov of the intrinsics (get_fov, all nine entries); campos = the
    rescaled translation; tanfov = tan(fov / 2) -- so that the full camera gradient reaches the extrinsics in all 16
    entries and the intrinsics in all 9, as that glue would carry it.  Off, the intrinsics get no gradient.  The CPU path
    is that glue in plain tensor code, differentiable throughout."""
    if extrinsics.is_cuda:
        return _make_view_batch_cuda(extrinsics, intrinsics, near, far, scale_invariant, camera_gradients)
    if scale_invariant:
        scale = 1.0 / near
        extrinsics = extrinsics.clone()
        extrinsics[..., :3, 3] = extrinsics[..., :3, 3] * scale[:, None]
        near = near * scale
        far = far * scale
    else:
        scale = torch.ones_like(near)
    fov = get_fov(intrinsics)
    fov_x, fov_y = fov.unbind(dim=-1)
    proj = get_projection_matrix(near, far, fov_x, fov_y).transpose(-1, -2)
    view = torch.linalg.inv(extrinsics).transpose(-1, -2)
    full = view @ proj
    tanfov = torch.stack(((0.5 * fov_x).tan(), (0.5 * fov_y).tan()), dim=-1)
    return ViewBatch(view.contiguous(), full.contiguous(), extrinsics[:, :3, 3].contiguous(), tanfov.contiguous(),
                     scale.contiguous())


def _make_view_batch_cuda(extrinsics, intrinsics, near, far, scale_invariant: bool, camera_gradients=None) -> ViewBatch:
    import ctypes

    from . import _capi
    dev = extrinsics.device
    B = extrinsics.shape[0]
    f = lambda t: t.detach().to(dev, torch.float32).contiguous()
    ext, intr, nr, fr = f(extrinsics), f(intrinsics), f(near), f(far)
    view = torch.empty(B, 4, 4, device=dev)
    proj = torch.empty(B, 4, 4, device=dev)
    campos = torch.empty(B, 3, device=dev)
    tanfov = torch.empty(B, 2, device=dev)
    scale = torch.empty(B, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    with torch.cuda.device(dev):
        _capi.check(_capi.lib().gs_view_batch(B, int(bool(scale_invariant)), p(ext), p(intr), p(nr), p(fr), p(view), p(proj),
                                              p(campos), p(tanfov), p(scale),
                                              ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    if camera_gradients is None:
        from .rasterizer import get_camera_gradients
        camera_gradients = get_camera_gradients()
    intr_grad = intrinsics.requires_grad
    if camera_gradients and (extrinsics.requires_grad or intr_grad) and torch.is_grad_enabled():
        # The kernel's values (plus exact zeros) with the gradients of render_cuda's glue (cuda_splatting.py:64-86)
        e = extrinsics.clone()
        inv_near = (1.0 / near.detach().to(dev, e.dtype))
        if scale_invariant:
            e[..., :3, 3] = e[..., :3, 3] * inv_near[:, None]
        vt = torch.linalg.inv(e).transpose(-1, -2)
        with torch.no_grad():
            nr_s, fr_s = (nr * scale, fr * scale) if scale_invariant else (nr, fr)
        # the intrinsics as given when they require grad, else the kernel's fp32 copy (no graph: P is a constant)
        fov_x, fov_y = get_fov(intrinsics.to(dev) if intr_grad else intr).unbind(-1)
        pt = get_projection_matrix(nr_s.to(fov_x.dtype), fr_s.to(fov_x.dtype), fov_x, fov_y).transpose(-1, -2).to(vt.dtype)
        full = vt @ pt
        cp = e[:, :3, 3]
        view = view + (vt - vt.detach()).to(view.dtype)
        proj = proj + (full - full.detach()).to(proj.dtype)
        campos = campos + (cp - cp.detach()).to(campos.dtype)
        if intr_grad:
            tan = torch.stack(((0.5 * fov_x).tan(), (0.5 * fov_y).tan()), dim=-1)
            tanfov = tanfov + (tan - tan.detach()).to(tanfov.dtype)
    elif extrinsics.requires_grad and torch.is_grad_enabled():
        # The kernel's values (plus exact zeros) with the gradient of a torch expression of the view matrix.  The
        # expression rescales the translation of extrinsics^-1 rather than that of the extrinsics
        # (cuda_splatting.py:64-86).  Both are equal while the bottom row is (0, 0, 0, 1), but only this one differentiates
        # like render_depth_cuda's z = (extrinsics^-1 @ mean).z once the depth is multiplied back by near, in every
        # entry, the bottom row's included.
        w2c = torch.linalg.inv(extrinsics).clone()
        if scale_invariant:
            w2c[..., :3, 3] = w2c[..., :3, 3] * (1.0 / near.detach().to(dev, w2c.dtype))[:, None]
        vt = w2c.transpose(-1, -2)
        view = view + (vt - vt.detach()).to(view.dtype)
    return ViewBatch(view, proj, campos, tanfov, scale)
