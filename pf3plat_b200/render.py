"""Batched render entry: the decoder-facing functions of the reference with the per-view Python loop, the v-fold
`repeat` of the Gaussians and the per-view host syncs removed (SURVEY.md section 8(f).1).

Replaces, behind the same argument meaning:
  * `render_cuda`        PF3plat's src/model/decoder/cuda_splatting.py:47-127
  * `render_depth_cuda`  PF3plat's src/model/decoder/cuda_splatting.py:226-269 (every DepthRenderingMode fused as a
                         4th composited channel; `render_depth` keeps the reference's second render to compare against)
  * the body of `DecoderSplattingCUDA.forward`  PF3plat's src/model/decoder/decoder_splatting_cuda.py:35-67
All views of all scenes go through ONE gs_forward call (one host sync per batch instead of three per view).
"""
from __future__ import annotations

from math import isqrt
from typing import Optional

import torch

from .cameras import make_view_batch
from .rasterizer import BatchSettings, rasterize_batch

_TRIU: dict = {}


def _cov6(cov: torch.Tensor) -> torch.Tensor:
    """(..., 3, 3) -> (..., 6) upper triangle in the order the call site uses (cuda_splatting.py:115,123).
    One gather forward and one index_add backward (the obvious stack of six slices costs ~25 small kernels per step)."""
    idx = _TRIU.get(cov.device)
    if idx is None:
        idx = _TRIU[cov.device] = torch.tensor([0, 1, 2, 4, 5, 8], device=cov.device)
    return torch.index_select(cov.flatten(-2), -1, idx)


def render_views(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                 gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities, scale_invariant: bool = True,
                 use_sh: bool = True, with_depth: bool = False, sh_layout: str = "g_xyz_n",
                 sh_eval_max_degree: Optional[int] = None, depth_mode: str = "depth", with_alpha: bool = False,
                 antialiasing: Optional[bool] = None, camera_gradients: Optional[bool] = None, workspace=None):
    """extrinsics (B,4,4) c2w, intrinsics (B,3,3), near/far (B,), background (B,3); Gaussians are per SCENE and NOT
    repeated per view: means (S,G,3), covariances (S,G,3,3) or (S,G,6), sh (S,G,3,d_sh) [or (S,G,d_sh,3) with
    sh_layout="g_n_xyz"], opacities (S,G); B % S == 0 and view b shows scene b // (B//S).
    sh_eval_max_degree: highest SH degree evaluated (3, or 4 for band 4 of d_sh = 25); None = the process-wide setting
    (rasterizer.set_sh_eval_max_degree, default 3).
    Returns color (B,3,h,w) and, if with_depth, depth (B,h,w) = sum_i alpha_i T_i f(z_i): f(z) = z of the (rescaled)
    scene for depth_mode "depth"; for "disparity", "relative_disparity" and "log" the fake colour of render_depth_cuda
    (cuda_splatting.py:245-251) at the UNSCALED camera-space depth z, with the unscaled near and far.
    with_alpha: also return the accumulated opacity alpha (B,h,w) = 1 - T_final, last: (color[, depth], alpha).
    antialiasing: the screen-space filter with opacity compensation (BatchSettings.antialiasing); None = the
    process-wide setting (rasterizer.set_antialiasing, default off).
    camera_gradients: extrinsics and intrinsics that require grad get the full gradient of every output (colour, depth,
    alpha, the anti-aliasing factor) through render_cuda's own camera glue (make_view_batch; the intrinsics through the
    fov, into tanfov and P); None = the process-wide setting (rasterizer.set_camera_gradients, default off: only the
    depth channel reaches the extrinsics, and the intrinsics get none).
    workspace: a rasterizer.SyncFreeWorkspace of this call's shape selects the sync-free path (rasterize_batch)."""
    assert use_sh or gaussian_sh_coefficients.shape[-1 if sh_layout == "g_xyz_n" else -2] == 1
    h, w = image_shape
    if camera_gradients is None:
        from .rasterizer import get_camera_gradients
        camera_gradients = get_camera_gradients()
    vb = make_view_batch(extrinsics, intrinsics, near, far, scale_invariant, camera_gradients)
    if sh_layout == "g_xyz_n":
        n = gaussian_sh_coefficients.shape[-1]
        shs = gaussian_sh_coefficients.transpose(-1, -2)  # (S,G,n,3); made contiguous by the operator
    else:
        n = gaussian_sh_coefficients.shape[-2]
        shs = gaussian_sh_coefficients
    degree = isqrt(n) - 1
    cov6 = gaussian_covariances if gaussian_covariances.shape[-1] == 6 and gaussian_covariances.dim() == 3 \
        else _cov6(gaussian_covariances)
    bs = BatchSettings(image_height=h, image_width=w, viewmatrix=vb.viewmatrix, projmatrix=vb.projmatrix,
                       campos=vb.campos, bg=background_color, sh_degree=degree, tanfov=vb.tanfov,
                       view_scale=vb.scale if scale_invariant else None, with_depth=with_depth,
                       sh_eval_max_degree=sh_eval_max_degree, depth_mode=depth_mode,
                       depth_near_far=torch.stack([near, far], -1) if with_depth and depth_mode != "depth" else None,
                       with_alpha=with_alpha, antialiasing=antialiasing, camera_gradients=bool(camera_gradients))
    B = extrinsics.shape[0]
    S = gaussian_means.shape[0]
    if use_sh:
        out = rasterize_batch(bs, gaussian_means, gaussian_opacities, shs=shs, cov3D_precomp=cov6, workspace=workspace)
    else:
        colors = shs[..., 0, :]                                  # (S,G,3)
        colors = colors.repeat_interleave(B // S, dim=0) if S != B else colors
        out = rasterize_batch(bs, gaussian_means, gaussian_opacities, colors_precomp=colors, cov3D_precomp=cov6,
                              workspace=workspace)
    if with_alpha:
        return (out[0], out[2], out[3]) if with_depth else (out[0], out[2])
    if with_depth:
        return out[0], out[2]
    return out[0]


def render_cuda(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities, scale_invariant: bool = True,
                use_sh: bool = True):
    """Signature-compatible with the reference's render_cuda (Gaussians already repeated per view: batch == views)."""
    return render_views(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                        gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities, scale_invariant, use_sh)


def decoder_forward(means, covariances, harmonics, opacities, extrinsics, intrinsics, near, far, image_shape,
                    background_color, depth_mode: Optional[str] = None, sh_eval_max_degree: Optional[int] = None,
                    return_alpha: bool = False, antialiasing: Optional[bool] = None,
                    camera_gradients: Optional[bool] = None, workspace=None):
    """`DecoderSplattingCUDA.forward` (decoder_splatting_cuda.py:35-67) without the v-fold repeat: Gaussians
    (b,g,...), cameras (b,v,...).  Returns (color (b,v,3,h,w), depth (b,v,h,w) or None).  Every depth_mode of the
    reference ("depth", "disparity", "relative_disparity", "log") is composited in the same pass as the colour.

    Gradients: like the reference's colour pass, the colour gives the CAMERAS no gradient.  The reference's depth
    pass builds its fake colour z = (extrinsics^-1 @ mean).z in torch (cuda_splatting.py:239-242), so its depth is
    differentiable w.r.t. the extrinsics -- PF3plat trains with depth_mode "depth" on predicted poses.  The fused
    channel gives exactly that gradient and no other: dL/ddepth reaches the z column of each view matrix through the
    mode's f'(z) (make_view_batch carries it on to the extrinsics), besides the Gaussians.  "log" clamps z as the
    reference does, to the constant log(far) when near < far: its extrinsics get a zero gradient.  A loss that does not
    read the depth leaves the extrinsics without a gradient, as the reference does.  So every mode is one render whether
    or not the extrinsics require grad.  sh_eval_max_degree: as render_views.
    return_alpha: also return the accumulated opacity (b,v,h,w) = 1 - T_final of the same pass, as (color, depth, alpha)
    (depth None without a depth_mode).  It trains the Gaussians' geometry and opacities, never the extrinsics.
    antialiasing: as render_views; the opacity compensation gives the extrinsics no gradient either.
    camera_gradients (None = rasterizer.get_camera_gradients(), default off): the extrinsics get the full gradient of
    every output instead -- colour, depth (the z-column route above is then part of it, not added again), alpha and
    the anti-aliasing factor -- for photometric pose training and test-time pose refinement; intrinsics that require
    grad get theirs too, in all nine entries (focal refinement, calibration-free use).
    workspace: a rasterizer.SyncFreeWorkspace for (b, b*v, g, image_shape) selects the sync-free path: the call never
    makes the host wait, so decoder, loss and backward can be captured in one CUDA graph (INTEGRATION.md)."""
    b, v = extrinsics.shape[:2]
    flat = lambda t: t.reshape(b * v, *t.shape[2:])
    bg = background_color.reshape(1, 3).expand(b * v, 3)
    out = render_views(flat(extrinsics), flat(intrinsics), flat(near), flat(far), image_shape, bg, means,
                       covariances, harmonics, opacities, with_depth=depth_mode is not None,
                       sh_eval_max_degree=sh_eval_max_degree, depth_mode=depth_mode or "depth", with_alpha=return_alpha,
                       antialiasing=antialiasing, camera_gradients=camera_gradients, workspace=workspace)
    alpha = None
    if return_alpha:
        *out, alpha = out
        out = out[0] if depth_mode is None else tuple(out)
        alpha = alpha.reshape(b, v, *alpha.shape[1:])
    if depth_mode is None:
        color = out.reshape(b, v, *out.shape[1:])
        return (color, None, alpha) if return_alpha else (color, None)
    color, depth = out
    if depth_mode == "depth":
        # the reference renders depth in the 1/near-rescaled scene (render_depth_cuda -> render_cuda with
        # scale_invariant=True) but takes the fake colour from the UNSCALED camera-space z
        # (cuda_splatting.py:239-242): undo the rescale of z (the other modes evaluate f at the unscaled z already)
        depth = depth * flat(near)[:, None, None]
    color, depth = color.reshape(b, v, *color.shape[1:]), depth.reshape(b, v, *depth.shape[1:])
    return (color, depth, alpha) if return_alpha else (color, depth)


def render_depth(means, covariances, opacities, extrinsics, intrinsics, near, far, image_shape, mode: str = "depth"):
    """`render_depth_cuda` (cuda_splatting.py:226-269) for (b,g,...) Gaussians and (b,v,...) cameras: a second render
    whose colour is the fake colour.  The reference's two-pass route for every mode, kept to compare the fused channel
    of `decoder_forward` against."""
    b, v = extrinsics.shape[:2]
    flat = lambda t: t.reshape(b * v, *t.shape[2:])
    ext, nr, fr = flat(extrinsics), flat(near), flat(far)
    w2c = torch.linalg.inv(ext)                                                   # (B,4,4)
    m = means.repeat_interleave(v, dim=0) if v > 1 else means                     # (B,g,3) view of scene per view
    z = torch.einsum("bj,bgj->bg", w2c[:, 2, :3], m) + w2c[:, 2, 3:4]
    if mode == "disparity":
        z = 1 / z
    elif mode == "relative_disparity":
        eps = 1e-10
        dn, df, d = 1 / (nr[:, None] + eps), 1 / (fr[:, None] + eps), 1 / (z + eps)
        z = 1 - (d - df) / (dn - df + eps)
    elif mode == "log":
        z = z.minimum(nr[:, None]).maximum(fr[:, None]).log()
    fake = z[..., None, None].expand(-1, -1, 3, 1)                                # (B,g,3,1)
    # fake colours are per VIEW, so this path needs Gaussians indexed per view: S == B
    cov = covariances.repeat_interleave(v, dim=0) if v > 1 else covariances
    opa = opacities.repeat_interleave(v, dim=0) if v > 1 else opacities
    out = render_views(ext, flat(intrinsics), nr, fr, image_shape, torch.zeros((b * v, 3), device=ext.device), m,
                       cov, fake, opa, use_sh=False)
    return out.mean(dim=1).reshape(b, v, *image_shape)
