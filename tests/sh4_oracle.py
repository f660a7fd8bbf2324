"""SH colour through band 4 on the CPU in fp64, and the batched rasterizer oracle at any SH degree up to 4.

The rasterizer's oracles (oracle/gs_oracle.c, oracle/torch_oracle.py) evaluate bands 0..3.  A render at SH degree d is,
view by view, the render of the precomputed colours rgb = max(sum_k sh_k Y_k(dir) + 0.5, 0) with dir the unit vector from
the camera to the (view-scaled) mean.  So the oracle at degree 4 is a composition:
  * forward: this module evaluates the SH colour of every (view, Gaussian) in fp64 and hands it to the batched oracle
    (`tests.batch_oracle.oracle_batch`) as colors_precomp;
  * backward: the oracle returns dL/dcolors per view; this module carries it, masked where the colour was clamped at 0,
    through the basis into dL/dSH and through the direction's normalisation into dL/dmeans3D.
The basis is the one the kernels use (gs_common.cuh): bands 0..3 as oracle/torch_oracle.py, band 4 continued with the same
Condon-Shortley signs, in the forms with "- 1" and "- 3" that hold on the unit sphere.  The partial derivatives of the basis
are taken by complex step (exact to rounding for polynomials), independently of the kernels' hand-written ones.
"""
from __future__ import annotations

import numpy as np
import torch

from tests.batch_oracle import _np, oracle_batch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435]
SH_C4 = [2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892, 0.10578554691520431,
         -0.6690465435572892, 0.47308734787878004, -1.7701307697799304, 0.6258357354491761]


def sh_basis(dirs, deg: int = 4):
    """(..., 3) unit directions (numpy, complex numpy or torch) -> (..., (deg+1)^2) basis values."""
    x, y, z = dirs[..., 0], dirs[..., 1], dirs[..., 2]
    one = x * 0 + 1
    out = [SH_C0 * one]
    if deg > 0:
        out += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        out += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
    if deg > 2:
        out += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4 * zz - xx - yy),
                SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
                SH_C3[6] * x * (xx - 3 * yy)]
    if deg > 3:
        out += [SH_C4[0] * xy * (xx - yy), SH_C4[1] * yz * (3 * xx - yy), SH_C4[2] * xy * (7 * zz - 1),
                SH_C4[3] * yz * (7 * zz - 3), SH_C4[4] * (zz * (35 * zz - 30) + 3), SH_C4[5] * xz * (7 * zz - 3),
                SH_C4[6] * (xx - yy) * (7 * zz - 1), SH_C4[7] * xz * (xx - 3 * yy),
                SH_C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))]
    if torch.is_tensor(dirs):
        return torch.stack(out, -1)
    return np.stack(out, -1)


def sh_basis_grad(dirs: np.ndarray, deg: int = 4) -> np.ndarray:
    """(..., 3) -> (..., (deg+1)^2, 3): d basis_k / d(x, y, z), x, y, z independent (complex step)."""
    h = 1e-30
    out = []
    for a in range(3):
        d = dirs.astype(np.complex128)
        d[..., a] += 1j * h
        out.append(sh_basis(d, deg).imag / h)
    return np.stack(out, -1)


def with_band4(scene, amplitude: float = 0.05, seed: int = 7):
    """The scene with random band-4 coefficients (harmonics[:, :, 16:25]) of the given scale (the synthetic scenes
    leave band 4 zero); d_sh must be >= 25."""
    import copy
    g = torch.Generator().manual_seed(seed)
    out = copy.copy(scene)
    h = scene.harmonics.clone()
    assert h.shape[-1] >= 25
    h[:, :, 16:25] = amplitude * torch.randn(h.shape[0], 3, 9, generator=g)
    out.harmonics = h.contiguous()
    return out


class ShOracleBatch:
    """`oracle_batch` of a call with shs [S,P,M,3], at SH degree `deg` (<= 4): see the module docstring."""

    def __init__(self, bs, means3D, opacities, shs, deg: int, scales=None, rotations=None, cov3D_precomp=None,
                 dtype=np.float64, frag_rel=1e-4):
        means = _np(means3D, np.float64)
        self.shs = _np(shs, np.float64)
        S, P, M = self.shs.shape[:3]
        self.deg = deg = min(int(deg), int(bs.sh_degree), int(np.sqrt(M)) - 1)
        self.K = (deg + 1) ** 2
        V = int(bs.viewmatrix.shape[0])
        self.S, self.P, self.M, self.V, self.VPS = S, P, M, V, V // S
        vs = np.ones(V) if bs.view_scale is None else _np(bs.view_scale, np.float64).reshape(V)
        self.s = vs.astype(np.float32).astype(np.float64)   # the kernels hold s in fp32
        campos = _np(bs.campos, np.float64).reshape(V, 3)
        cols, self.dirs, self.dlen, self.clamped = [], [], [], []
        for v in range(V):
            k = v // self.VPS
            d = means[k] * self.s[v] - campos[v]
            n = np.linalg.norm(d, axis=-1, keepdims=True)
            u = d / n
            raw = np.einsum("pk,pkc->pc", sh_basis(u, deg), self.shs[k, :, :self.K]) + 0.5
            cols.append(np.maximum(raw, 0.0))
            self.dirs.append(u)
            self.dlen.append(n)
            self.clamped.append(raw < 0)
        self.colors = np.stack(cols)
        self.batch = oracle_batch(bs, means3D, opacities, colors_precomp=self.colors.astype(dtype), scales=scales,
                                  rotations=rotations, cov3D_precomp=cov3D_precomp, dtype=dtype, frag_rel=frag_rel)

    @property
    def color(self):
        return self.batch.color

    @property
    def depth(self):
        return self.batch.depth

    @property
    def radii(self):
        return self.batch.radii

    def affected(self):
        return self.batch.affected()

    def backward(self, dL_dcolor, dL_ddepth=None) -> dict:
        g = self.batch.backward(dL_dcolor, dL_ddepth)
        gsh = np.zeros((self.S, self.P, self.M, 3))
        for v in range(self.V):
            k, s = v // self.VPS, self.s[v]
            gc = np.where(self.clamped[v], 0.0, g["colors_precomp"][v])                  # [P,3]
            u = self.dirs[v]
            gsh[k, :, :self.K] += sh_basis(u, self.deg)[:, :, None] * gc[:, None, :]
            ddir = np.einsum("pka,pkc,pc->pa", sh_basis_grad(u, self.deg), self.shs[k, :, :self.K], gc)
            dd = (ddir - u * np.sum(u * ddir, -1, keepdims=True)) / self.dlen[v]   # through d / |d|
            g["means3D"][k] += s * dd
        g["shs"] = gsh
        g["colors_precomp"] = None
        return g


SH_BANDS4 = [("band0", slice(0, 1)), ("band1", slice(1, 4)), ("band2", slice(4, 9)), ("band3", slice(9, 16)),
             ("band4", slice(16, 25))]
