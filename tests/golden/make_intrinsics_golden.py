"""Generates tests/golden/intrinsics_glue.npz: the intrinsics' share of the REFERENCE's own render_cuda glue, in fp64 under
autograd.  PF3plat's get_fov (src/geometry/projection.py:233-247), get_projection_matrix and render_cuda
(src/model/decoder/cuda_splatting.py:17-87) run unmodified, imported from a PF3plat checkout as make_camera_golden.py does,
against a recording stand-in for `diff_gaussian_rasterization` that keeps the autograd graph of the full projection it is
handed.  Their float32 constants and buffers are read as float64 (the modules see a `torch` whose float32 is float64), so
the fixture is the glue's exact arithmetic at double precision.

Recorded per view, for the scale-invariant ("si") and the raw glue: tanfov = tan(fov / 2), the projection P
(get_projection_matrix, untransposed) and the full projection render_cuda hands its rasterizer (transposed), each with
the vector-Jacobian product of a seeded cotangent with respect to all nine entries of the intrinsics.  The cameras
have off-centre principal points, unequal fx and fy and a small skew, all of which change the fov.
Usage: PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_intrinsics_golden.py"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_camera_golden as mcg  # noqa: E402

RECORDED: list = []


class _GraphRecorder:
    def __init__(self, raster_settings):
        self.s = raster_settings

    def __call__(self, means3D, means2D, **kw):
        RECORDED.append(self.s.projmatrix)
        return torch.zeros(3, self.s.image_height, self.s.image_width), torch.zeros(means3D.shape[0], dtype=torch.int32)


class _Torch64(types.ModuleType):
    """torch, with float32 read as float64."""

    def __getattr__(self, name):
        return torch.float64 if name == "float32" else getattr(torch, name)


def make_cameras(seed, B):
    ext, intr, near, far = (t.double() for t in mcg.make_cameras(seed, B))
    g = torch.Generator().manual_seed(seed + 1)
    intr[:, 0, 2] = 0.5 + 0.1 * torch.randn(B, generator=g, dtype=torch.float64)
    intr[:, 1, 2] = 0.5 + 0.1 * torch.randn(B, generator=g, dtype=torch.float64)
    intr[:, 0, 1] = 0.02 * torch.randn(B, generator=g, dtype=torch.float64)
    return ext, intr, near, far


def main():
    mod = mcg.load_reference_render_cuda()
    mod.GaussianRasterizer = _GraphRecorder
    proj_mod = sys.modules["src.geometry.projection"]
    mod.torch = proj_mod.torch = _Torch64("torch")
    B, G = 7, 2
    ext, intr, near, far = make_cameras(41, B)
    g = torch.Generator().manual_seed(42)
    means = torch.randn(B, G, 3, generator=g, dtype=torch.float64)
    a = torch.randn(B, G, 3, 3, generator=g, dtype=torch.float64)
    cov = a @ a.transpose(-1, -2)
    sh = torch.randn(B, G, 3, 4, generator=g, dtype=torch.float64)
    opac = torch.rand(B, G, generator=g, dtype=torch.float64)
    cot = dict(tanfov=torch.randn(B, 2, generator=g, dtype=torch.float64),
               P=torch.randn(B, 4, 4, generator=g, dtype=torch.float64),
               full=torch.randn(B, 4, 4, generator=g, dtype=torch.float64))
    arrays = dict(extrinsics=ext.numpy(), intrinsics=intr.numpy(), near=near.numpy(), far=far.numpy(),
                  **{f"cot_{k}": t.numpy() for k, t in cot.items()})
    for tag, si in (("si", True), ("raw", False)):
        K = intr.clone().requires_grad_(True)
        fov_x, fov_y = proj_mod.get_fov(K).unbind(-1)
        tanfov = torch.stack(((0.5 * fov_x).tan(), (0.5 * fov_y).tan()), -1)
        nr, fr = (near * (1 / near), far * (1 / near)) if si else (near, far)   # render_cuda's own rescale (:64-71)
        P = mod.get_projection_matrix(nr, fr, fov_x, fov_y)
        RECORDED.clear()
        mod.render_cuda(ext, K, near, far, (16, 24), torch.zeros(B, 3, dtype=torch.float64), means, cov, sh, opac,
                        scale_invariant=si)
        assert len(RECORDED) == B
        full = torch.stack(RECORDED)
        for k, t in (("tanfov", tanfov), ("P", P), ("full", full)):
            assert t.dtype == torch.float64, (k, t.dtype)
            arrays[f"{tag}_{k}"] = t.detach().numpy()
            arrays[f"{tag}_vjp_{k}"] = torch.autograd.grad((t * cot[k]).sum(), K, retain_graph=True)[0].numpy()
    RECORDED.clear()
    path = os.path.join(HERE, "intrinsics_glue.npz")
    np.savez_compressed(path, **arrays)
    print({k: v.shape for k, v in arrays.items()}, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
