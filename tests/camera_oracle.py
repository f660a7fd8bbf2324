"""Camera gradient (gs_backward_cam) from the fp64 autograd oracle, by composition.

oracle/torch_oracle.py renders one view in fp64 with every input a torch tensor, so handing it viewmatrix, projmatrix and
campos as leaves that require grad differentiates the whole forward -- projection, covariance, SH direction, depth,
tile membership masks aside -- with respect to the cameras.  The features it does not draw itself are composed around
it, each as the kernels define it:
  * view_scale s: the view-scaled scene (means * s, cov3D * s^2 or scales * s) is what the view is drawn from;
  * anti-aliasing: opacities o * rho_v, rho from a differentiable restatement of the projected covariance that reads the
    view-matrix leaf (tests/aa_oracle.py's projection, here on the leaf);
  * a depth mode other than "depth": a second render of the same view whose colour is f(z) at the unscaled z (z from the
    view-matrix leaf) on a black background, channel 0;
  * alpha: a render with colour 1 on black, channel 0;
  * SH degree 4: the colour max(sum_k sh_k Y_k(dir) + 0.5, 0) evaluated here through band 4 (tests/sh4_oracle.py's basis)
    with dir from the campos leaf, handed over as colors_precomp.
This is autograd of the fp64 torch restatement rather than a chain of oracle/gs_oracle.c's screen-space gradients: the
C oracle does not expose dL/dconic or dL/dz.  The restatement follows the same conventions (clamped t.x / t.y detached,
the 0.99 clamp passed straight through) and tests/test_camera_grad_cpu.py pins it to central finite differences.
The loss <dL, colour> + <w, depth> + <dA, alpha> is differentiated by autograd; the leaves' .grad are the camera gradient
in the layouts of GsCameraGrads."""
from __future__ import annotations

import dataclasses

import numpy as np
import torch

from oracle.torch_oracle import render
from tests.aa_oracle import aa_ratio, aa_rho, sigma3
from tests.batch_oracle import _np, batch_view_settings
from tests.sh4_oracle import sh_basis


def cov2d_leaf(st, view, means, Sigma):
    """(a0, b, c0) of view settings `st` with the (4,4) transposed view matrix `view` (a tensor, maybe a leaf)."""
    P = means.shape[0]
    p_view = torch.cat([means, torch.ones(P, 1, dtype=means.dtype)], -1) @ view
    tz = p_view[:, 2]
    limx, limy = st.guard_band * st.tanfovx, st.guard_band * st.tanfovy
    txtz, tytz = p_view[:, 0] / tz, p_view[:, 1] / tz
    inx, iny = (txtz >= -limx) & (txtz <= limx), (tytz >= -limy) & (tytz <= limy)
    tx = torch.where(inx, p_view[:, 0], (txtz.clamp(-limx, limx) * tz).detach())
    ty = torch.where(iny, p_view[:, 1], (tytz.clamp(-limy, limy) * tz).detach())
    fx, fy = st.image_width / (2 * st.tanfovx), st.image_height / (2 * st.tanfovy)
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -fx * tx / (tz * tz), zero, fy / tz, -fy * ty / (tz * tz)], -1).reshape(P, 2, 3)
    Mm = J @ view[:3, :3].T
    cov = Mm @ Sigma @ Mm.transpose(-1, -2)
    return cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]


def depth_f(mode, z, near, far):
    """render_depth_cuda's fake colour of a depth mode at the unscaled z (pf3plat_b200.render.render_depth)."""
    if mode == "disparity":
        return 1 / z
    if mode == "relative_disparity":
        eps = 1e-10
        dn, df, d = 1 / (near + eps), 1 / (far + eps), 1 / (z + eps)
        return 1 - (d - df) / (dn - df + eps)
    if mode == "log":
        return z.minimum(torch.as_tensor(near, dtype=z.dtype)).maximum(torch.as_tensor(far, dtype=z.dtype)).log()
    raise ValueError(mode)


def camera_oracle(bs, ins, dL, w=None, dA=None, antialiasing=False, depth_mode="depth", near_far=None):
    """bs: BatchSettings (CPU tensors); ins: the Gaussian inputs of rasterize_batch; dL [V,3,H,W], w [V,H,W] or None,
    dA [V,H,W] or None.  Returns (dL/dviewmatrix [V,16], dL/dprojmatrix [V,16], dL/dcampos [V,3]) in fp64 numpy."""
    V = int(bs.viewmatrix.shape[0])
    out = [np.zeros((V, 16)), np.zeros((V, 16)), np.zeros((V, 3))]
    for v in range(V):
        loss, leaves = view_loss(bs, ins, v, dL, w, dA, antialiasing, depth_mode, near_far)
        loss.backward()
        for j in range(3):   # (campos: no grad without SH)
            if leaves[j].grad is not None:
                out[j][v] = leaves[j].grad.reshape(-1).numpy()
    return tuple(out)


def view_loss(bs, ins, v, dL, w=None, dA=None, antialiasing=False, depth_mode="depth", near_far=None):
    """The fp64 loss of view v, <dL, colour> + <w, depth> + <dA, alpha>, and its camera leaves (viewmatrix [16],
    projmatrix [16], campos [3])."""
    V = int(bs.viewmatrix.shape[0])
    t64 = lambda x: None if x is None else torch.as_tensor(_np(x, np.float64))
    I = {k: t64(x) for k, x in ins.items()}
    S = I["means3D"].shape[0]
    VPS = V // S
    M = 0 if I.get("shs") is None else I["shs"].shape[2]
    vs = np.ones(V) if bs.view_scale is None else _np(bs.view_scale, np.float64).reshape(V).astype(np.float32)
    k, s = v // VPS, float(vs[v])
    st0 = batch_view_settings(bs, v, M)
    leaves = [torch.as_tensor(np.asarray(x, np.float64)).reshape(-1).clone().requires_grad_(True)
              for x in (st0.viewmatrix, st0.projmatrix, st0.campos)]
    view, proj, campos = leaves[0].reshape(4, 4), leaves[1].reshape(4, 4), leaves[2].reshape(3)
    st = dataclasses.replace(st0, viewmatrix=view, projmatrix=proj, campos=campos)
    black = dataclasses.replace(st, bg=np.zeros(3))
    means = I["means3D"][k] * s
    Sig = sigma3(I, k, float(bs.scale_modifier)) * (s * s)
    c = Sig.reshape(-1, 9)
    geo = {"cov3D_precomp": torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 4], c[:, 5], c[:, 8]], -1)}
    opac = I["opacities"][k].reshape(-1)
    if antialiasing:
        a0, b, c0 = cov2d_leaf(st, view, means, Sig)
        opac = opac * aa_rho(aa_ratio(a0, b, c0, st.dilation))
    if I.get("shs") is None:
        col = {"colors_precomp": I["colors_precomp"][v]}
    elif min(st0.sh_degree, bs.sh_eval_max_degree or 3) >= 4:
        d = means - campos
        rgb = (sh_basis(d / d.norm(dim=-1, keepdim=True), 4)[..., None] * I["shs"][k][:, :25]).sum(1) + 0.5
        col = {"colors_precomp": torch.clamp_min(rgb, 0.0)}
    else:
        col = {"shs": I["shs"][k]}
    color, _, depth = render(st, means, opac, **col, **geo, with_depth=True)
    loss = (color * t64(dL)[v]).sum()
    if w is not None:
        if depth_mode == "depth":
            loss = loss + (depth * t64(w)[v]).sum()
        else:
            P = means.shape[0]
            z = (torch.cat([means, torch.ones(P, 1, dtype=means.dtype)], -1) @ view)[:, 2] / s
            nf = _np(near_far, np.float64)[v] if near_far is not None else (0.0, 0.0)
            fz = depth_f(depth_mode, z, float(nf[0]), float(nf[1]))
            dimg = render(black, means, opac, colors_precomp=fz[:, None].expand(-1, 3), **geo)[0][0]
            loss = loss + (dimg * t64(w)[v]).sum()
    if dA is not None:
        ones = torch.ones(means.shape[0], 3, dtype=means.dtype)
        aimg = render(black, means, opac, colors_precomp=ones, **geo)[0][0]
        loss = loss + (aimg * t64(dA)[v]).sum()
    return loss, leaves
