"""fp64 restatement of PF3plat's plane-sweep cost volume (depth_predictor_multiview.py:91-141 and :309-343, the tensor
before the torch.cat), with grid_sample's bilinear taps written out.  Differentiable with respect to `features` by
torch autograd; it runs on whatever device its inputs are on.

Each step is the reference's, in the reference's order:
  * views in (v b) order; for source slot s = 1 .. v-1 the source of view vi is (vi + s) mod v;
  * the relative pose E[v1]^-1 E[v0] (v > 2), or for v = 2 pose = E[1]^-1 E[0] and cat(pose, pose^-1);
  * the TARGET view's intrinsics, row 0 times w and row 1 times h (skew and principal point included);
  * depth candidates 1 / (1/far + linspace(0, 1, D) (1/near - 1/far));
  * pixel-index coordinates (no +0.5), points = K (R (K^-1 p) z + t), divided by clamp(z, min=1e-3);
  * bilinear sampling with align_corners=True (the sample coordinate is the pixel coordinate itself): taps (x0, y0),
    (x0+1, y0), (x0, y0+1), (x0+1, y0+1) with x0 = floor(x), each multiplied in when in bounds, whatever its weight, and
    zero otherwise (zero padding per tap);
  * sum over C of feat01 * warped, / sqrt(C), then the mean over the v - 1 sources.
"""
from __future__ import annotations

import torch


def relative_poses(extrinsics: torch.Tensor) -> list:
    """-> [v-1] tensors [(v b), 4, 4]: the pose of source slot s = 1 .. v-1 for every target, in (v b) order."""
    b, v = extrinsics.shape[:2]
    E = extrinsics
    if v == 2:
        pose = torch.linalg.inv(E[:, 1]) @ E[:, 0]
        return [torch.cat((pose, torch.linalg.inv(pose)), dim=0)]
    out = []
    for s in range(1, v):
        out.append(torch.cat([torch.linalg.inv(E[:, (vi + s) % v]) @ E[:, vi] for vi in range(v)], dim=0))
    return out


def unnormalised_intrinsics(intrinsics: torch.Tensor, h: int, w: int) -> torch.Tensor:
    K = intrinsics[..., :3, :3].clone()
    K[..., 0, :] *= float(w)
    K[..., 1, :] *= float(h)
    b, v = K.shape[:2]
    return K.transpose(0, 1).reshape(v * b, 3, 3)


def depth_candidates(near: torch.Tensor, far: torch.Tensor, D: int) -> torch.Tensor:
    """[(v b), D]"""
    lo = (1.0 / far).transpose(0, 1).reshape(-1, 1)
    hi = (1.0 / near).transpose(0, 1).reshape(-1, 1)
    t = torch.linspace(0.0, 1.0, D, dtype=lo.dtype, device=lo.device)[None]
    return 1.0 / (lo + t * (hi - lo))


def sample_coordinates(K, pose, depth, h, w):
    """pixel coordinates (ix, iy), each [(v b), D, h*w], of every target pixel at every candidate depth"""
    nv = K.shape[0]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=K.dtype, device=K.device),
                            torch.arange(w, dtype=K.dtype, device=K.device), indexing="ij")
    grid = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(h * w, dtype=K.dtype, device=K.device)])  # [3, hw]
    pts = torch.linalg.inv(K) @ grid  # [nv, 3, hw]
    pts = (pose[:, :3, :3] @ pts)[:, :, None, :] * depth[:, None, :, None]  # [nv, 3, D, hw]
    pts = pts + pose[:, :3, 3][:, :, None, None]
    pts = (K @ pts.reshape(nv, 3, -1)).reshape(nv, 3, depth.shape[1], h * w)
    z = pts[:, 2].clamp(min=1e-3)
    return pts[:, 0] / z, pts[:, 1] / z


def bilinear(src: torch.Tensor, ix: torch.Tensor, iy: torch.Tensor) -> torch.Tensor:
    """src [n, C, h, w]; ix, iy [n, D, hw] -> warped [n, C, D, hw]: grid_sample(bilinear, zeros, align_corners=True)."""
    n, C, h, w = src.shape
    flat = src.reshape(n, C, h * w)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    x1, y1 = x0 + 1, y0 + 1
    taps = ((x0, y0, (x1 - ix) * (y1 - iy)), (x1, y0, (ix - x0) * (y1 - iy)),
            (x0, y1, (x1 - ix) * (iy - y0)), (x1, y1, (ix - x0) * (iy - y0)))
    out = torch.zeros((n, C) + tuple(ix.shape[1:]), dtype=src.dtype, device=src.device)
    for tx, ty, wt in taps:
        inb = (tx >= 0) & (tx <= w - 1) & (ty >= 0) & (ty <= h - 1)
        idx = torch.where(inb, ty * w + tx, torch.zeros_like(tx)).long().reshape(n, 1, -1).expand(n, C, -1)
        val = torch.gather(flat, 2, idx).reshape(out.shape)
        out = out + torch.where(inb[:, None], val * wt[:, None], torch.zeros((), dtype=src.dtype, device=src.device))
    return out


def cost_volume(features, intrinsics, extrinsics, near, far, D: int) -> torch.Tensor:
    """-> [(v b), D, h, w], the dtype of `features` (pass float64 inputs for the oracle)."""
    b, v, C, h, w = features.shape
    with torch.no_grad():
        K = unnormalised_intrinsics(intrinsics.detach(), h, w)
        depth = depth_candidates(near.detach(), far.detach(), D)
        coords = [sample_coordinates(K, pose, depth, h, w) for pose in relative_poses(extrinsics.detach())]
    feat01 = features.transpose(0, 1).reshape(v * b, C, h * w)
    total = 0
    for s, (ix, iy) in enumerate(coords, start=1):
        order = [(vi + s) % v for vi in range(v)]
        feat10 = features[:, order].transpose(0, 1).reshape(v * b, C, h, w)
        warped = bilinear(feat10, ix, iy)  # [vb, C, D, hw]
        total = total + (feat01[:, :, None, :] * warped).sum(1) / C ** 0.5
    return (total / (v - 1)).reshape(v * b, D, h, w)
