"""PF3plat's depth rendering modes (DepthRenderingMode, cuda_splatting.py:223-251) restated in fp64, and the oracle of the
reference's construction of the depth image for a batched call.

`fake_depth` is the fake colour render_depth_cuda builds from the UNSCALED camera-space depth z of each mean and the
unscaled near / far of the view (relative disparity: depth_to_relative_disparity of conversions.py:17-27, in its own
expression order); `fake_depth_grad` is its derivative in z.  tests/test_depth_modes_cpu.py pins both to the reference's
recorded fake colours and to torch autograd.

`depth_mode_oracle` renders what the reference renders: `tests.batch_oracle.oracle_batch` with colors_precomp = f(z) on a
black background, the mean over the three channels.  Its colour gradient per (view, Gaussian) is dL/df; times
f'(z) dz/dz_s it is the gradient of the view-scaled depth z_s = (view matrix z column) . (s mean, 1), which the oracle
carries on into the means and into the z column of each view matrix (generalising `view_z_oracle` of
tests/test_gpu_pose_depth.py).  The colour image is a second oracle render with the call's own colours."""
from __future__ import annotations

import numpy as np

from tests.batch_oracle import oracle_batch

MODES = ("disparity", "relative_disparity", "log")
EPS = 1e-10


def fake_depth(mode, z, near, far):
    z = np.asarray(z, np.float64)
    if mode == "depth":
        return z
    if mode == "disparity":
        return 1 / z
    if mode == "relative_disparity":
        dn, df, d = 1 / (near + EPS), 1 / (far + EPS), 1 / (z + EPS)
        return 1 - (d - df) / (dn - df + EPS)
    if mode == "log":
        return np.log(np.maximum(np.minimum(z, near), far))
    raise ValueError(mode)


def fake_depth_grad(mode, z, near, far):
    z = np.asarray(z, np.float64)
    if mode == "depth":
        return np.ones_like(z)
    if mode == "disparity":
        return -1 / (z * z)
    if mode == "relative_disparity":
        return 1 / ((z + EPS) ** 2 * (1 / (near + EPS) - 1 / (far + EPS) + EPS))
    if mode == "log":   # 1/z where z passes both clamps: nowhere when near < far
        near, far = np.broadcast_to(near, z.shape), np.broadcast_to(far, z.shape)
        return np.where((z < near) & (z > far), 1 / z, 0.0)
    raise ValueError(mode)


class DepthModeOracle:
    """bs: BatchSettings with CPU tensors; ins: the Gaussian inputs of rasterize_batch (CPU); mode; near_far (V,2).
    Images: `color` [V,3,H,W], `depth` [V,H,W], `frag` [V,H,W] (fragile depth pixels).  `backward(dL_dcolor, w)` returns
    the gradients of <dL_dcolor, colour> + <w, depth>: the Gaussian inputs' (per scene, as rasterize_batch returns them),
    and `view_z` [V,4] = dL/d(view matrix flat entries 2, 6, 10, 14) with its per-Gaussian terms `view_z_terms` [V,P,4]."""

    def __init__(self, bs, ins, mode, near_far):
        V = bs.viewmatrix.shape[0]
        means = ins["means3D"].double().cpu().numpy()
        S, P = means.shape[:2]
        self.S, self.P, self.V, self.VPS, self.mode = S, P, V, V // S, mode
        self.s = bs.view_scale.cpu().numpy().astype(np.float32).astype(np.float64)   # held in fp32, as the kernels do
        self.vm = bs.viewmatrix.double().cpu().numpy()                                # transposed: [:, :, 2] is the z column
        self.hom = np.concatenate([means[np.arange(V) // self.VPS] * self.s[:, None, None], np.ones((V, P, 1))], -1)
        zs = np.einsum("vpj,vj->vp", self.hom, self.vm[:, :, 2])
        nf = np.asarray(near_far.cpu() if hasattr(near_far, "cpu") else near_far, np.float64)
        self.near, self.far = nf[:, :1], nf[:, 1:]
        self.z = zs / self.s[:, None]                       # the reference's unscaled camera-space depth
        self.f = fake_depth(mode, self.z, self.near, self.far)
        geo = {k: v for k, v in ins.items() if k not in ("shs", "colors_precomp")}
        import torch
        self.ob_depth = oracle_batch(bs._replace(bg=torch.zeros(V, 3, dtype=torch.float64), with_depth=False),
                                     colors_precomp=np.repeat(self.f[..., None], 3, -1), dtype=np.float64, **geo)
        self.ob_color = oracle_batch(bs._replace(with_depth=False), dtype=np.float64, **ins)
        self.color = self.ob_color.color
        self.depth = self.ob_depth.color.mean(axis=1)
        self.frag = np.stack([r.px_fragile for r in self.ob_depth.views])
        self.frag_color = np.stack([r.px_fragile for r in self.ob_color.views])

    def affected(self) -> np.ndarray:
        return self.ob_color.affected() | self.ob_depth.affected()

    def affected_views(self) -> np.ndarray:
        return np.repeat(self.affected(), self.VPS, axis=0)

    def backward(self, dL_dcolor, w) -> dict:
        g = self.ob_color.backward(dL_dcolor)
        gd = self.ob_depth.backward(np.repeat(np.asarray(w, np.float64)[:, None] / 3.0, 3, axis=1))
        for k in ("means3D", "means2D", "opacities", "scales", "rotations", "cov3D_precomp"):
            if g[k] is not None:
                g[k] = g[k] + gd[k]
        # dL/dz_s per (view, Gaussian): the fake colour's gradient through f'(z) dz/dz_s
        gzs = gd["colors_precomp"].sum(-1) * fake_depth_grad(self.mode, self.z, self.near, self.far) / self.s[:, None]
        for v in range(self.V):
            g["means3D"][v // self.VPS] += (gzs[v] * self.s[v])[:, None] * self.vm[v, :3, 2][None]
        g["view_z_terms"] = gzs[..., None] * self.hom
        g["view_z"] = g["view_z_terms"].sum(axis=1)
        g["z_path"] = gzs
        return g
