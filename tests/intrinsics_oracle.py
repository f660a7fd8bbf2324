"""Intrinsics gradient (gs_backward_cam_tanfov's dL/dtanfov) from the fp64 autograd oracle, by composition.

tests/camera_oracle.py differentiates oracle/torch_oracle.py's forward with the view matrix, the full projection and
campos as leaves.  This is the same loss with tanfov [2] as a fourth leaf, handed to the oracle as the settings'
tanfovx / tanfovy, so autograd follows it into the focal lengths of the projection Jacobian, fx = W / (2 tanfovx) and
fy = H / (2 tanfovy) -- in every render of the loss (colour, f(z) depth, alpha) and in the anti-aliasing factor.

One term needs composing: the oracle detaches a guard-band-clamped t.x (it is a constant with respect to the view
matrix), but t.x = +-guard_band tanfovx t.z still moves with tanfovx, and with it J02 = -fx t.x / t.z^2 does not: fx t.x
is W guard_band t.z / 2 for every tanfovx.  Autograd of the oracle sees J02 through fx only, d J02 / d tanfovx = -J02 /
tanfovx, so for each clamped Gaussian the composition adds +J02 / tanfovx through a zero-valued scalar delta placed on
J02: the covariance handed to the oracle is A Sigma A^T with A = I + delta_x u_x r^T + delta_y u_y r^T, where r is the
third column of the view rotation and M u_x = e_0, M u_y = e_1 for the oracle's M = J W.  Then (M A) Sigma (M A)^T is
the 2-D covariance with J02 + delta_x and J12 + delta_y.  delta is exactly 0, so A = I and the forward is the camera
oracle's, bit for bit; only its derivative, (tanfov - tanfov.detach()) J02 / tanfovx, carries the term.
tests/test_intrinsics_grad_cpu.py pins the result to central finite differences in tanfov, clamped Gaussians included."""
from __future__ import annotations

import dataclasses

import numpy as np
import torch

from oracle.torch_oracle import render
from tests.aa_oracle import aa_ratio, aa_rho, sigma3
from tests.batch_oracle import _np, batch_view_settings
from tests.camera_oracle import cov2d_leaf, depth_f
from tests.sh4_oracle import sh_basis


def clamp_compensated_sigma(st, view, tan, means, Sig):
    """Sigma [P,3,3] of the view-scaled means, as A Sigma A^T (see the module docstring): equal in value, with the
    guard-band clamp's tanfov derivative on J02 / J12 of the Gaussians it clamps."""
    with torch.no_grad():
        P = means.shape[0]
        W = view.detach()
        p_view = torch.cat([means.detach(), torch.ones(P, 1, dtype=means.dtype)], -1) @ W
        tz = p_view[:, 2]
        tx_, ty_ = float(tan[0]), float(tan[1])
        limx, limy = st.guard_band * tx_, st.guard_band * ty_
        txtz, tytz = p_view[:, 0] / tz, p_view[:, 1] / tz
        inx, iny = (txtz >= -limx) & (txtz <= limx), (tytz >= -limy) & (tytz <= limy)
        tx, ty = txtz.clamp(-limx, limx) * tz, tytz.clamp(-limy, limy) * tz
        fx, fy = st.image_width / (2 * tx_), st.image_height / (2 * ty_)
        zero = torch.zeros_like(tz)
        J = torch.stack([fx / tz, zero, -fx * tx / (tz * tz), zero, fy / tz, -fy * ty / (tz * tz)], -1).reshape(P, 2, 3)
        M = J @ W[:3, :3].T
        U = M.transpose(-1, -2) @ torch.linalg.inv(M @ M.transpose(-1, -2))   # [P,3,2]: M U = I
        r = W[:3, 2]
        kx = torch.where(inx, zero, J[:, 0, 2] / tx_)
        ky = torch.where(iny, zero, J[:, 1, 2] / ty_)
    dx = (tan[0] - tan[0].detach()) * kx
    dy = (tan[1] - tan[1].detach()) * ky
    A = torch.eye(3, dtype=Sig.dtype) + (dx[:, None, None] * U[:, :, 0:1] + dy[:, None, None] * U[:, :, 1:2]) * r[None, None, :]
    return A @ Sig @ A.transpose(-1, -2)


def intrinsics_view_loss(bs, ins, v, dL, w=None, dA=None, antialiasing=False, depth_mode="depth", near_far=None):
    """tests/camera_oracle.view_loss with tanfov as a fourth leaf: the fp64 loss of view v and its leaves (viewmatrix
    [16], projmatrix [16], campos [3], tanfov [2])."""
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
              for x in (st0.viewmatrix, st0.projmatrix, st0.campos, (st0.tanfovx, st0.tanfovy))]
    view, proj, campos, tan = leaves[0].reshape(4, 4), leaves[1].reshape(4, 4), leaves[2].reshape(3), leaves[3]
    st = dataclasses.replace(st0, viewmatrix=view, projmatrix=proj, campos=campos, tanfovx=tan[0], tanfovy=tan[1])
    black = dataclasses.replace(st, bg=np.zeros(3))
    means = I["means3D"][k] * s
    Sig = clamp_compensated_sigma(st, view, tan, means, sigma3(I, k, float(bs.scale_modifier)) * (s * s))
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


def intrinsics_oracle(bs, ins, dL, w=None, dA=None, antialiasing=False, depth_mode="depth", near_far=None):
    """As tests/camera_oracle.camera_oracle, plus dL/dtanfov: returns (dL/dviewmatrix [V,16], dL/dprojmatrix [V,16],
    dL/dcampos [V,3], dL/dtanfov [V,2]) in fp64 numpy.  bs.tanfov (V,2) or bs.tanfovx / tanfovy give the values."""
    V = int(bs.viewmatrix.shape[0])
    out = [np.zeros((V, 16)), np.zeros((V, 16)), np.zeros((V, 3)), np.zeros((V, 2))]
    for v in range(V):
        loss, leaves = intrinsics_view_loss(bs, ins, v, dL, w, dA, antialiasing, depth_mode, near_far)
        loss.backward()
        for j in range(4):
            if leaves[j].grad is not None:
                out[j][v] = leaves[j].grad.reshape(-1).numpy()
    return tuple(out)


def clamped_pairs(bs, ins, v):
    """Number of Gaussians of view v whose t.x or t.y the guard band clamps (so a test can show it covers them)."""
    V = int(bs.viewmatrix.shape[0])
    S = int(torch.as_tensor(_np(ins["means3D"])).shape[0])
    M = 0 if ins.get("shs") is None else int(ins["shs"].shape[2])
    st = batch_view_settings(bs, v, M)
    s = 1.0 if bs.view_scale is None else float(_np(bs.view_scale, np.float64).reshape(V).astype(np.float32)[v])
    m = torch.as_tensor(_np(ins["means3D"], np.float64))[v // (V // S)] * s
    p = torch.cat([m, torch.ones(m.shape[0], 1, dtype=m.dtype)], -1) @ torch.as_tensor(np.asarray(st.viewmatrix)).reshape(4, 4)
    out_x = (p[:, 0] / p[:, 2]).abs() > st.guard_band * st.tanfovx
    out_y = (p[:, 1] / p[:, 2]).abs() > st.guard_band * st.tanfovy
    return int((out_x | out_y).sum())
