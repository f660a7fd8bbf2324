"""Rotation of real spherical-harmonics coefficients (mirror of PF3plat's src/misc/sh_rotation.py:10-36).

The reference builds one Wigner-D matrix per degree with `e3nn.o3.wigner_D(degree, *matrix_to_angles(R))` and applies
it to the coefficients of that degree.  e3nn is a third-party dependency that is absent from this image
(PF3plat's requirements.txt lists it unpinned).  This module therefore

* uses e3nn exactly as the reference does when it is importable, and otherwise
* derives the same matrices from their defining property  Y_l(R x) = D_l(R) Y_l(x)  by a least-squares fit over a
  fixed set of unit vectors, with e3nn's real basis RESTATED FROM ITS PUBLISHED DEFINITION (parity unpinned): the
  orthonormal real harmonics without Condon-Shortley phase, polar axis y, i.e. the standard z-polar polynomials
  evaluated at (x_std, y_std, z_std) = (z, x, y); for degree 1 that is the (x, y, z) order and D_1(R) = R.

The fused adapter kernel (pf3plat_b200/adapter.py) takes the block-diagonal matrix as an input, so a caller who has
e3nn (or any other convention) can always supply its own.  `guarded_sh_rotation_blocks` builds that matrix on the
device, guard included, with the same fit (csrc/gs_sh_rotation.cu); the tensor functions here stay the CPU path and
the reference it is checked against.
"""
from __future__ import annotations

import ctypes
from math import isqrt

import torch

try:  # pragma: no cover - not installed in this image
    from e3nn.o3 import matrix_to_angles as _e3nn_angles, wigner_D as _e3nn_wigner_D
    HAVE_E3NN = True
except Exception:  # ImportError and whatever a broken install raises
    HAVE_E3NN = False


def real_sh_basis(degree: int, xyz: torch.Tensor) -> torch.Tensor:
    """(..., 3) unit vectors -> (..., 2*degree+1) orthonormal real harmonics in e3nn's component order."""
    x, y, z = xyz[..., 2], xyz[..., 0], xyz[..., 1]  # standard (z-polar) polynomials at (z, x, y)
    xx, yy, zz = x * x, y * y, z * z
    if degree == 0:
        out = [0.28209479177387814 * torch.ones_like(x)]
    elif degree == 1:
        c = 0.4886025119029199
        out = [c * y, c * z, c * x]
    elif degree == 2:
        out = [1.0925484305920792 * x * y, 1.0925484305920792 * y * z, 0.31539156525252005 * (2 * zz - xx - yy),
               1.0925484305920792 * x * z, 0.5462742152960396 * (xx - yy)]
    elif degree == 3:
        out = [0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * y * z,
               0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
               0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
               0.5900435899266435 * x * (xx - 3 * yy)]
    elif degree == 4:
        rr = xx + yy + zz
        out = [2.5033429417967046 * x * y * (xx - yy), 1.7701307697799304 * y * z * (3 * xx - yy),
               0.9461746957575601 * x * y * (7 * zz - rr), 0.6690465435572892 * y * z * (7 * zz - 3 * rr),
               0.10578554691520431 * (35 * zz * zz - 30 * zz * rr + 3 * rr * rr),
               0.6690465435572892 * x * z * (7 * zz - 3 * rr), 0.47308734787878004 * (xx - yy) * (7 * zz - rr),
               1.7701307697799304 * x * z * (xx - 3 * yy), 0.6258357354491761 * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))]
    else:
        raise ValueError("real_sh_basis: degree <= 4")
    return torch.stack(out, dim=-1)


_FIT_CACHE: dict = {}


def _fit_points(degree: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    key = (degree, str(device))
    if key not in _FIT_CACHE:
        g = torch.Generator().manual_seed(1234 + degree)
        pts = torch.randn(64, 3, generator=g, dtype=torch.float64)
        pts = (pts / pts.norm(dim=-1, keepdim=True)).to(device)
        pinv = torch.linalg.pinv(real_sh_basis(degree, pts).T)  # (64, 2l+1): Y(X)^+ with Y(X) of shape (2l+1, 64)
        _FIT_CACHE[key] = (pts, pinv)
    return _FIT_CACHE[key]


def wigner_d_from_matrix(degree: int, rotations: torch.Tensor) -> torch.Tensor:
    """(..., 3, 3) proper rotations -> (..., 2l+1, 2l+1) with Y_l(R x) = D Y_l(x)."""
    if HAVE_E3NN:  # the reference's own route
        alpha, beta, gamma = _e3nn_angles(rotations)
        return _e3nn_wigner_D(degree, alpha, beta, gamma).to(rotations.dtype)
    pts, pinv = _fit_points(degree, rotations.device)
    rot = rotations.to(torch.float64)
    moved = torch.einsum("...ij,kj->...ki", rot, pts)            # R x_k
    yr = real_sh_basis(degree, moved).transpose(-1, -2)           # (..., 2l+1, 64)
    return (yr @ pinv).to(rotations.dtype)


def sh_rotation_blocks(rotations: torch.Tensor, d_sh: int) -> torch.Tensor:
    """Block-diagonal (..., d_sh, d_sh) matrix holding D_0 .. D_{sqrt(d_sh)-1}: what the adapter kernel consumes."""
    out = torch.zeros(*rotations.shape[:-2], d_sh, d_sh, dtype=rotations.dtype, device=rotations.device)
    for degree in range(isqrt(d_sh)):
        lo, hi = degree ** 2, (degree + 1) ** 2
        out[..., lo:hi, lo:hi] = wigner_d_from_matrix(degree, rotations)
    return out


def rotations_are_proper(rotations: torch.Tensor) -> bool:
    """The reference's guard (sh_rotation.py:21): every determinant allclose to 1, else ALL rotations -> identity."""
    return bool(torch.allclose(torch.det(rotations), rotations.new_tensor(1)))


def guarded_sh_rotation_blocks(rotations: torch.Tensor, d_sh: int) -> torch.Tensor:
    """The block-diagonal (..., d_sh, d_sh) matrices of sh_rotation_blocks after the reference's all-or-nothing guard
    (rotate_sh's rotations_are_proper: unless every determinant is allclose to 1, every rotation of the call is the
    identity), on the device (csrc/gs_sh_rotation.cu): two launches, no host synchronisation, the same least-squares fit
    in fp64 from the same fit points, rounded to float32 once.

    rotations: float32 CUDA [..., 3, 3], or [..., 4, 4] whose top-left 3 x 3 block is the rotation (c2w itself).  Up to
    two batch dims are read in place with any strides, so c2w[:, ::V - 1] costs no gather; more are reshaped.  Not
    differentiable (the reference detaches the rotation, gaussian_adapter.py:81): inputs that require grad are
    refused."""
    from . import _capi
    if not torch.is_tensor(rotations):
        raise TypeError("guarded_sh_rotation_blocks: rotations must be a tensor")
    if rotations.device.type != "cuda":
        raise TypeError(f"guarded_sh_rotation_blocks: rotations must be a CUDA tensor (the tensor route "
                        f"sh_rotation_blocks is the CPU path), got {rotations.device}")
    if rotations.dtype != torch.float32:
        raise TypeError(f"guarded_sh_rotation_blocks: rotations must be float32, got {rotations.dtype}")
    if rotations.requires_grad:
        raise ValueError("guarded_sh_rotation_blocks is not differentiable: pass rotations.detach() (the reference "
                         "detaches the rotation, gaussian_adapter.py:81)")
    if not isinstance(d_sh, int) or isinstance(d_sh, bool) or d_sh not in (1, 4, 9, 16, 25):
        raise ValueError(f"guarded_sh_rotation_blocks: d_sh must be 1, 4, 9, 16 or 25, got {d_sh!r}")
    if rotations.dim() < 2 or tuple(rotations.shape[-2:]) not in ((3, 3), (4, 4)):
        raise ValueError(f"guarded_sh_rotation_blocks needs [..., 3, 3] or [..., 4, 4] rotations, got "
                         f"{tuple(rotations.shape)}")
    batch = rotations.shape[:-2]
    out = torch.empty(*batch, d_sh, d_sh, dtype=torch.float32, device=rotations.device)
    if out.numel() == 0:
        return out
    r = rotations if len(batch) <= 2 else rotations.reshape(-1, *rotations.shape[-2:])
    if r.stride(-1) != 1 or r.stride(-2) not in (3, 4):
        r = r.contiguous()
    lead = (1,) * (2 - (r.dim() - 2)) + tuple(r.shape[:-2])
    strides = (0,) * (2 - (r.dim() - 2)) + tuple(r.stride()[:-2])
    cfg = _capi.GsShRotationConfig(outer=lead[0], inner=lead[1], outer_stride=strides[0], inner_stride=strides[1],
                                   row_stride=r.stride(-2), d_sh=d_sh)
    L = _capi.lib()
    workspace = torch.empty(max(L.gs_sh_rotation_workspace_bytes(ctypes.byref(cfg)), 16), dtype=torch.uint8,
                            device=r.device)
    with torch.cuda.device(r.device):
        stream = ctypes.c_void_p(torch.cuda.current_stream(r.device).cuda_stream)
        _capi.check(L.gs_sh_rotation_blocks(ctypes.byref(cfg), ctypes.c_void_p(r.data_ptr()),
                                            ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(workspace.data_ptr()),
                                            stream))
    return out


def rotate_sh(sh_coefficients: torch.Tensor, rotations: torch.Tensor) -> torch.Tensor:
    """Same signature and behaviour as the reference's rotate_sh (sh_rotation.py:10-36)."""
    n = sh_coefficients.shape[-1]
    if not rotations_are_proper(rotations):
        rotations = torch.eye(3, device=rotations.device, dtype=rotations.dtype).expand(rotations.shape[:-2] + (3, 3))
    result = []
    for degree in range(isqrt(n)):
        d = wigner_d_from_matrix(degree, rotations).to(sh_coefficients.dtype)
        result.append(torch.einsum("...ij,...j->...i", d, sh_coefficients[..., degree ** 2:(degree + 1) ** 2]))
    return torch.cat(result, dim=-1)
