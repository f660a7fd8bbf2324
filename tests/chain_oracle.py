"""The differentiable chain PF3plat trains through -- Gaussian adapter -> batched decoder (`decoder_forward`) -> colour and
depth -- restated on the CPU in fp64 by composing the two oracles that already exist: `oracle.adapter_oracle` (torch
autograd) and `tests.batch_oracle.oracle_batch` (the rasterizer's CPU oracle, one render per view).

The glue between them is laid out exactly as `pf3plat_b200.render` lays it out:
  * one scene per batch element, the context views' Gaussians flattened into the Gaussian axis;
  * harmonics (b, G, 3, d_sh) handed over transposed, as (b, G, d_sh, 3);
  * the covariance's upper triangle gathered in the order [0, 1, 2, 4, 5, 8] of the flattened (3, 3) matrix by
    `index_select`, so that its backward scatters the six gradients into an upper-triangular (3, 3) gradient;
  * target cameras from `make_view_batch` (view_scale = 1/near); the fused depth channel multiplied by `near`.
When the target extrinsics carry a gradient, `decoder_forward` takes the reference's two-pass route instead: the depth is a
second render whose colour is the camera-space z of each Gaussian, computed in torch from the extrinsics (as
`tests.ref_callsite.render_depth_like_reference` does), so that dL/dz reaches the extrinsics through dL/dcolors_precomp.

Per-camera gradients (context c2w, K^-1 through the intrinsics, target extrinsics) are sums over thousands of Gaussians.
To bound them where a Gaussian sits at a fragile decision, the camera tensors enter the oracle expanded per Gaussian; the
`.grad` of the expanded tensor is each Gaussian's contribution, and the camera gradient is its sum (`camera_grad_check`).
"""
from __future__ import annotations

from math import isqrt

import numpy as np
import torch

from oracle import adapter_oracle
from pf3plat_b200.cameras import make_view_batch
from pf3plat_b200.rasterizer import BatchSettings
from pf3plat_b200.sh_rotation import rotations_are_proper, sh_rotation_blocks
from tests.batch_oracle import oracle_batch

TRIU = torch.tensor([0, 1, 2, 4, 5, 8])


def _np(t):
    return t.detach().cpu().numpy()


def target_settings(extrinsics, intrinsics, near, far, image_shape, background, sh_degree, with_depth) -> BatchSettings:
    """BatchSettings of the b*v target views as `decoder_forward` builds them (cameras detached), in fp64."""
    B = extrinsics.shape[0] * extrinsics.shape[1]
    f = lambda t: t.detach().double().cpu().reshape(B, *t.shape[2:])
    vb = make_view_batch(f(extrinsics), f(intrinsics), f(near), f(far), scale_invariant=True)
    bg = torch.as_tensor(background).detach().double().cpu().reshape(1, 3).expand(B, 3).contiguous()
    return BatchSettings(image_height=image_shape[0], image_width=image_shape[1], viewmatrix=vb.viewmatrix,
                         projmatrix=vb.projmatrix, campos=vb.campos, bg=bg, sh_degree=sh_degree, tanfov=vb.tanfov,
                         view_scale=vb.scale, with_depth=with_depth)


class DecoderOracle:
    """`decoder_forward(..., depth_mode="depth")` on fp64 torch tensors: means (b,G,3), covariances (b,G,3,3), harmonics
    (b,G,3,d_sh), opacities (b,G); target extrinsics (b,v,4,4), intrinsics (b,v,3,3), near / far (b,v), background (3,).

    two_pass=False: one render with the fused depth channel (depth * near).  two_pass=True: colour render plus the
    fake-colour depth render.  `z_extrinsics` (two-pass only) is what the fake colour z is computed from: (b,v,4,4), or
    (b,v,G,4,4) to get per-Gaussian contributions to the extrinsics' gradient; by default `extrinsics`.  The rasterized
    cameras always come from `extrinsics`, detached, as in `decoder_forward`.

    `color` (b*v,3,H,W) and `depth` (b*v,H,W) are numpy; `backward(dL_dcolor, dL_ddepth)` runs the oracles' backward and
    carries it through torch autograd into whatever the input tensors were computed from."""

    def __init__(self, means, covariances, harmonics, opacities, extrinsics, intrinsics, near, far, image_shape, background,
                 two_pass=False, z_extrinsics=None, frag_rel=1e-4):
        b, v = extrinsics.shape[:2]
        self.b, self.v, self.two_pass = b, v, two_pass
        cov6 = torch.index_select(covariances.flatten(-2), -1, TRIU)
        shs = harmonics.transpose(-1, -2)
        deg = isqrt(shs.shape[-2]) - 1
        self.near = _np(near).reshape(-1).astype(np.float64)
        bs = target_settings(extrinsics, intrinsics, near, far, image_shape, background, deg, with_depth=not two_pass)
        self.ob = oracle_batch(bs, _np(means), _np(opacities), shs=_np(shs), cov3D_precomp=_np(cov6), dtype=np.float64,
                               frag_rel=frag_rel)
        self._outs = [means, cov6, shs, opacities]
        self.color = self.ob.color
        if not two_pass:
            self.depth = self.ob.depth * self.near[:, None, None]
            self.ob_depth = None
            return
        # render_depth_like_reference: z in the UNSCALED camera of each view, rendered as a grey colour on a black
        # background, averaged over the three channels
        ze = extrinsics if z_extrinsics is None else z_extrinsics
        hom = torch.cat([means, torch.ones_like(means[..., :1])], dim=-1).repeat_interleave(v, dim=0)     # (b*v,G,4)
        if ze.dim() == 4:
            cam = torch.einsum("bij,bgj->bgi", ze.reshape(b * v, 4, 4).inverse(), hom)
        else:
            cam = torch.einsum("bgij,bgj->bgi", ze.reshape(b * v, *ze.shape[2:]).inverse(), hom)
        fake = cam[..., 2]
        colors = fake[..., None].expand(-1, -1, 3)
        bs_d = bs._replace(bg=torch.zeros_like(bs.bg))
        self.ob_depth = oracle_batch(bs_d, _np(means), _np(opacities), colors_precomp=_np(colors),
                                     cov3D_precomp=_np(cov6), dtype=np.float64, frag_rel=frag_rel)
        self.depth = self.ob_depth.color.mean(axis=1)
        self._fake = fake

    def affected(self) -> np.ndarray:
        """bool[b, G]: the Gaussians at a fragile decision in any render of their scene."""
        aff = self.ob.affected()
        if self.ob_depth is not None:
            aff |= self.ob_depth.affected()
        return aff

    def raster_grads(self, dL_dcolor, dL_ddepth=None) -> dict:
        """The oracle's gradients at the rasterizer's inputs (numpy, summed over each scene's views): means3D, opacities,
        shs, cov3D_precomp, and in the two-pass route the per-view fake colour z."""
        dLc = np.asarray(dL_dcolor, np.float64)
        if not self.two_pass:
            dLd = None if dL_ddepth is None else np.asarray(dL_ddepth, np.float64) * self.near[:, None, None]
            return self.ob.backward(dLc, dLd)
        g = self.ob.backward(dLc)
        out = {k: g[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
        out["fake"] = np.zeros(self._fake.shape)
        if dL_ddepth is not None:
            dLd = np.asarray(dL_ddepth, np.float64)
            gd = self.ob_depth.backward(np.repeat(dLd[:, None] / 3.0, 3, axis=1))
            for k in ("means3D", "opacities", "cov3D_precomp"):
                out[k] = out[k] + gd[k]
            out["fake"] = gd["colors_precomp"].sum(axis=-1)
        return out

    def backward(self, dL_dcolor, dL_ddepth=None) -> dict:
        g = self.raster_grads(dL_dcolor, dL_ddepth)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
        outs, grads = [], []
        for o, k in zip(self._outs, ("means3D", "cov3D_precomp", "shs", "opacities")):
            if o.requires_grad:
                outs.append(o)
                grads.append(t(g[k]).reshape(o.shape))
        if self.two_pass and self._fake.requires_grad:
            outs.append(self._fake)
            grads.append(t(g["fake"]))
        if outs:
            torch.autograd.backward(outs, grads)
        return g


def default_sh_rotation(extrinsics, d_sh):
    """What GaussianAdapter does without an explicit sh_rotation: Wigner-D blocks of the (detached) c2w rotation, or the
    identity (None) for d_sh == 1 or improper rotations."""
    rot = extrinsics[..., :3, :3].detach().double()
    if d_sh == 1 or not rotations_are_proper(rot.reshape(-1, 3, 3)):
        return None
    return sh_rotation_blocks(rot.reshape(-1, 3, 3), d_sh).reshape(*rot.shape[:-2], d_sh, d_sh)


class ChainOracle:
    """Adapter -> decoder in fp64.  Context inputs per scene and context view: extrinsics (b,vc,4,4), intrinsics
    (b,vc,3,3), coordinates (b,vc,R,2), depths (b,vc,R), opacities (b,vc,R), raw_gaussians (b,vc,R,7+3*d_sh); targets as
    `DecoderOracle`.  The leaves (fp64 copies, `self.leaves`) get their gradients from `backward`; `self.leaves` holds
    extrinsics / intrinsics expanded per Gaussian (b,vc,R,...) and "target_extrinsics" expanded (b,vt,G,4,4) in the
    two-pass route, so their .grad are per-Gaussian contributions; `grads()` sums them per camera."""

    def __init__(self, extrinsics, intrinsics, coordinates, depths, opacities, raw_gaussians, context_shape, sh_degree,
                 target_extrinsics, target_intrinsics, near, far, image_shape, background, two_pass=False,
                 scale_min=0.5, scale_max=15.0, frag_rel=1e-4):
        d64 = lambda t: torch.as_tensor(t).detach().double().cpu()
        b, vc, R = depths.shape
        self.b, self.vc, self.R = b, vc, R
        d_sh = (sh_degree + 1) ** 2
        L = {"extrinsics": d64(extrinsics)[:, :, None].expand(b, vc, R, 4, 4).clone(),
             "intrinsics": d64(intrinsics)[:, :, None].expand(b, vc, R, 3, 3).clone(),
             "coordinates": d64(coordinates).clone(), "depths": d64(depths).clone(),
             "opacities": d64(opacities).clone(), "raw_gaussians": d64(raw_gaussians).clone()}
        for k, t in L.items():
            t.requires_grad_(True)
        D = default_sh_rotation(d64(extrinsics), d_sh)
        o = adapter_oracle.adapter_forward(L["extrinsics"], L["intrinsics"], L["coordinates"], L["depths"],
                                           L["opacities"], L["raw_gaussians"], context_shape, sh_degree, scale_min,
                                           scale_max, sh_rotation=None if D is None else D[:, :, None])
        G = vc * R
        means = o["means"].reshape(b, G, 3)
        cov = o["covariances"].reshape(b, G, 3, 3)
        harm = o["harmonics"].reshape(b, G, 3, d_sh)
        opac = o["opacities"].reshape(b, G)
        tgt = d64(target_extrinsics)
        z_ext = None
        if two_pass:
            vt = tgt.shape[1]
            L["target_extrinsics"] = z_ext = tgt[:, :, None].expand(b, vt, G, 4, 4).clone().requires_grad_(True)
        self.leaves = L
        self.adapter_out = o
        self.decoder = DecoderOracle(means, cov, harm, opac, tgt, d64(target_intrinsics), d64(near), d64(far),
                                     image_shape, d64(background), two_pass=two_pass, z_extrinsics=z_ext,
                                     frag_rel=frag_rel)
        self.color, self.depth = self.decoder.color, self.decoder.depth

    def backward(self, dL_dcolor, dL_ddepth=None):
        self.decoder.backward(dL_dcolor, dL_ddepth)

    def affected(self) -> np.ndarray:
        """bool[b, vc, R]: the fragile Gaussians of `DecoderOracle.affected`, in the adapter's layout."""
        return self.decoder.affected().reshape(self.b, self.vc, self.R)

    def grads(self) -> dict:
        """Gradients at the chain's inputs, per camera where the input is per camera (contributions summed)."""
        L = self.leaves
        g = {k: L[k].grad for k in ("coordinates", "depths", "opacities", "raw_gaussians")}
        g["extrinsics"] = L["extrinsics"].grad.sum(dim=2)
        g["intrinsics"] = L["intrinsics"].grad.sum(dim=2)
        if "target_extrinsics" in L:
            g["target_extrinsics"] = L["target_extrinsics"].grad.sum(dim=2)
        return g

    def contributions(self, name) -> torch.Tensor:
        """Per-Gaussian contributions (cameras..., Gaussians, ...) to the camera gradient `name`."""
        return self.leaves[name].grad


def nearby_poses(g: torch.Generator, base: torch.Tensor, n: int, angle: float, shift: float) -> torch.Tensor:
    """(b,4,4) c2w -> (b,n,4,4): each base pose turned by `angle` radians about a random axis and moved by up to `shift`
    in its own frame, so that every pose sees roughly what the base pose sees."""
    b = base.shape[0]
    axis = torch.randn(b, n, 3, generator=g, dtype=torch.float64)
    axis = axis / axis.norm(dim=-1, keepdim=True) * angle
    K = torch.zeros(b, n, 3, 3, dtype=torch.float64)
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -axis[..., 2], axis[..., 1], -axis[..., 0]
    K = K - K.transpose(-1, -2)
    delta = torch.eye(4, dtype=torch.float64).repeat(b, n, 1, 1)
    delta[..., :3, :3] = torch.linalg.matrix_exp(K)
    delta[..., :3, 3] = shift * (2 * torch.rand(b, n, 3, generator=g, dtype=torch.float64) - 1)
    return (base.double()[:, None] @ delta).float()


def make_chain_inputs(seed, b, vc, hw_context, vt, sh_degree, near):
    """Seeded adapter -> decoder inputs shaped as PF3plat's encoder hands them over: context views turned a few degrees
    from a random proper pose per scene, Gaussians 1 .. 10 units along the context pixels' rays (the adapter golden
    generator's distribution), target views turned ~8 degrees from the same pose, normalised intrinsics."""
    import os
    import sys
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    if golden not in sys.path:
        sys.path.insert(0, golden)
    import make_adapter_golden as mk
    h, w = hw_context
    R = h * w
    inp = mk.make_inputs(seed, b, vc, h, w, sh_degree)
    g = torch.Generator().manual_seed(seed + 500)
    base = mk.random_pose(g, b)
    ctx = nearby_poses(g, base, vc, 0.05, 0.05)
    tgt = nearby_poses(g, base, vt, 0.14, 0.1)
    tin = torch.eye(3).repeat(b, vt, 1, 1)
    tin[..., 0, 0] = 0.8 + 0.2 * torch.rand(b, vt, generator=g)
    tin[..., 1, 1] = 0.8 + 0.2 * torch.rand(b, vt, generator=g)
    tin[..., 0, 2] = tin[..., 1, 2] = 0.5
    return dict(extrinsics=ctx, intrinsics=inp["intrinsics"].reshape(b, vc, 3, 3),
                coordinates=inp["coordinates"].reshape(b, vc, R, 2), depths=inp["depths"].reshape(b, vc, R),
                opacities=inp["opacities"].reshape(b, vc, R), raw_gaussians=inp["raw_gaussians"].reshape(b, vc, R, -1),
                target_extrinsics=tgt, target_intrinsics=tin, near=torch.full((b, vt), float(near)),
                far=torch.full((b, vt), 100.0))


def camera_grad_check(label, got, ref, contrib, affected, rtol=1e-3, rtol_affected=1e-2) -> dict:
    """A gradient that is a sum over Gaussians, per camera: got / ref (cams..., *shape), contrib (cams..., N, *shape) the
    oracle's per-Gaussian terms, affected bool (cams..., N).  The element-wise rule of tests.util carried through the sum:
    |got - ref| <= rtol (|ref| + rms(ref)) + rtol_affected * sum over the affected Gaussians of |contribution|."""
    got = np.asarray(got.detach().cpu() if torch.is_tensor(got) else got, np.float64)
    ref = np.asarray(ref, np.float64).reshape(got.shape)
    c = np.abs(np.asarray(contrib, np.float64))
    nc = np.ndim(affected) - 1            # number of camera dims
    aff = np.asarray(affected, bool).reshape(c.shape[:nc + 1] + (1,) * (c.ndim - nc - 1))
    slack = (c * aff).sum(axis=nc)
    rms = float(np.sqrt(np.mean(ref * ref)))
    err = np.abs(got - ref)
    tol = rtol * (np.abs(ref) + rms) + rtol_affected * slack
    rep = {"name": label, "elements": int(ref.size), "rms": rms, "max_err": float(err.max()),
           "worst_ratio": float((err / (np.abs(ref) + rms + 1e-300)).max()),
           "worst_err_over_tol": float((err / (tol + 1e-300)).max()),
           "affected_gaussians": int(np.asarray(affected).sum())}
    print(f"[parity] camera grad {rep}")
    assert (err <= tol).all(), rep
    return rep
