"""The batched operator (`pf3plat_b200.rasterizer.rasterize_batch`: V views of S scenes per call) restated as one CPU oracle
render per view, so that every input the batched entry takes -- several views per scene, per-view `colors_precomp`,
scales + rotations with a scale modifier, the per-view 1/near rescale `view_scale` -- is checked against an independent
implementation rather than against another GPU path.

View v shows scene v // (V / S).  The 1/near rescale is applied to the oracle's inputs the way the kernels apply it
(include/gsplat_b200.h, GsConfig.view_scale): means * s, cov3D * s^2, scales * s, each multiplication carried out in the
oracle's own precision.  The backward undoes it by the chain rule (* s for means and scales, * s^2 for cov3D) and sums the
per-scene gradients over the views of each scene, as the kernels do.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.gs_oracle import OracleRender, OracleSettings


def _np(t, dtype=None):
    if t is None:
        return None
    a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    return a if dtype is None else a.astype(dtype)


def batch_view_settings(bs, v: int, M: int) -> OracleSettings:
    """OracleSettings of view v of a BatchSettings.  The SH degree is the one the operator evaluates: sh_degree, but
    never more bands than the M coefficients supplied hold."""
    tan = (float(bs.tanfovx), float(bs.tanfovy)) if bs.tanfov is None else tuple(float(x) for x in _np(bs.tanfov[v]))
    deg = int(bs.sh_degree)
    if M > 0:
        deg = min(deg, math.isqrt(M) - 1)
    return OracleSettings(
        image_height=int(bs.image_height), image_width=int(bs.image_width), tanfovx=tan[0], tanfovy=tan[1],
        bg=_np(bs.bg[v], np.float64), scale_modifier=float(bs.scale_modifier), viewmatrix=_np(bs.viewmatrix[v], np.float64),
        projmatrix=_np(bs.projmatrix[v], np.float64), sh_degree=deg, campos=_np(bs.campos[v], np.float64),
        prefiltered=bool(bs.prefiltered))


class OracleBatch:
    """One OracleRender per view of a batched call; see `oracle_batch`."""

    def __init__(self, bs, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                 cov3D_precomp=None, dtype=np.float32, frag_rel=1e-4):
        dt = np.dtype(dtype)
        self.dtype = dt
        means3D = _np(means3D, dt)
        S, P = means3D.shape[:2]
        V = int(bs.viewmatrix.shape[0])
        assert V % S == 0, (V, S)
        self.S, self.P, self.V, self.VPS = S, P, V, V // S
        opac = _np(opacities, dt).reshape(S, P)
        shs, colors_precomp = _np(shs, dt), _np(colors_precomp, dt)
        scales, rotations, cov3D = _np(scales, dt), _np(rotations, dt), _np(cov3D_precomp, dt)
        self.M = 0 if shs is None else shs.shape[2]
        vs = np.ones(V) if bs.view_scale is None else _np(bs.view_scale, np.float64).reshape(V)
        # the kernels hold s (and s^2) in fp32
        self.s = vs.astype(np.float32).astype(dt)
        self.with_depth = bool(bs.with_depth)
        self.views: list[OracleRender] = []
        for v in range(V):
            k = v // self.VPS
            s = self.s[v]
            kw = {"means3D": means3D[k] * s, "opacities": opac[k]}
            if shs is not None:
                kw["shs"] = shs[k]
            else:
                kw["colors_precomp"] = colors_precomp[v]
            if cov3D is not None:
                kw["cov3D_precomp"] = cov3D[k] * (s * s)
            else:
                kw["scales"] = scales[k] * s
                kw["rotations"] = rotations[k]
            self.views.append(OracleRender(batch_view_settings(bs, v, self.M), dtype=dt, with_depth=self.with_depth,
                                           frag_rel=frag_rel, **kw))
        self.has_sh = shs is not None
        self.has_scales = scales is not None

    @property
    def color(self) -> np.ndarray:
        return np.stack([r.color for r in self.views])

    @property
    def depth(self) -> np.ndarray:
        return np.stack([r.depth for r in self.views])

    @property
    def radii(self) -> np.ndarray:
        return np.stack([r.radii for r in self.views])

    def affected(self) -> np.ndarray:
        """bool[S, P]: per scene, the Gaussians that touch a fragile pixel or sit at a fragile geometric decision in any of
        the scene's views (the `affected` argument of tests.util.check_grad)."""
        from tests.util import affected_gaussians
        out = np.zeros((self.S, self.P), bool)
        for v, r in enumerate(self.views):
            out[v // self.VPS] |= affected_gaussians(r, r.px_fragile) | r.geom_fragile
        return out

    def backward(self, dL_dcolor, dL_ddepth=None) -> dict:
        """dL_dcolor [V,3,H,W], dL_ddepth [V,H,W] or None.  Returns the gradients `rasterize_batch` returns: per scene
        (summed over the scene's views, view-scale chain rule applied) means3D [S,P,3], opacities [S,P], shs [S,P,M,3],
        scales [S,P,3], rotations [S,P,4], cov3D_precomp [S,P,6]; per view means2D [V,P,3], colors_precomp [V,P,3]."""
        S, P, V, dt = self.S, self.P, self.V, np.float64
        g = {"means3D": np.zeros((S, P, 3), dt), "opacities": np.zeros((S, P), dt), "means2D": np.zeros((V, P, 3), dt),
             "shs": np.zeros((S, P, self.M, 3), dt) if self.has_sh else None,
             "colors_precomp": None if self.has_sh else np.zeros((V, P, 3), dt),
             "scales": np.zeros((S, P, 3), dt) if self.has_scales else None,
             "rotations": np.zeros((S, P, 4), dt) if self.has_scales else None,
             "cov3D_precomp": None if self.has_scales else np.zeros((S, P, 6), dt)}
        dLc = _np(dL_dcolor, self.dtype)
        dLd = _np(dL_ddepth, self.dtype)
        for v, r in enumerate(self.views):
            k, s = v // self.VPS, float(self.s[v])
            gv = r.backward(dLc[v], None if dLd is None else dLd[v])
            g["means3D"][k] += s * gv["means3D"]
            g["opacities"][k] += gv["opacities"][:, 0]
            g["means2D"][v] = gv["means2D"]
            if self.has_sh:
                g["shs"][k] += gv["shs"]
            else:
                g["colors_precomp"][v] = gv["colors_precomp"]
            if self.has_scales:
                g["scales"][k] += s * gv["scales"]
                g["rotations"][k] += gv["rotations"]
            else:
                g["cov3D_precomp"][k] += (s * s) * gv["cov3D_precomp"]
        return g


def oracle_batch(bs, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
                 dtype=np.float32, frag_rel=1e-4) -> OracleBatch:
    """Takes exactly what `rasterize_batch` takes (tensors on any device, or arrays): means3D [S,P,3], opacities [S,P] or
    [S,P,1], shs [S,P,M,3] | colors_precomp [V,P,3], scales [S,P,3] + rotations [S,P,4] | cov3D_precomp [S,P,6]."""
    return OracleBatch(bs, means3D, opacities, shs=shs, colors_precomp=colors_precomp, scales=scales, rotations=rotations,
                       cov3D_precomp=cov3D_precomp, dtype=dtype, frag_rel=frag_rel)


def scene_batch_args(scenes, views_per_scene=None, near=None, use_sh=True, device="cpu"):
    """(BatchSettings fields, inputs) for S synthetic scenes rendered through their own cameras, through the camera glue of
    the reference call site (pf3plat_b200.cameras.make_view_batch, with the 1/near rescale).  `near` [V] overrides the
    scenes' near planes (view_scale = 1/near)."""
    from pf3plat_b200.cameras import make_view_batch
    cat = lambda name: torch.cat([getattr(sc, name) for sc in scenes])
    ext, intr = cat("extrinsics"), cat("intrinsics")
    nr = cat("near") if near is None else torch.as_tensor(near, dtype=torch.float32)
    vb = make_view_batch(ext, intr, nr, cat("far"), scale_invariant=True)
    cams = {"viewmatrix": vb.viewmatrix, "projmatrix": vb.projmatrix, "campos": vb.campos, "tanfov": vb.tanfov,
            "view_scale": vb.scale, "bg": cat("background")}
    cams = {k: v.float().contiguous().to(device) for k, v in cams.items()}
    cov6 = lambda c: torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], -1)
    stack = lambda f: torch.stack([f(sc) for sc in scenes]).float().contiguous().to(device)
    ins = {"means3D": stack(lambda sc: sc.means), "opacities": stack(lambda sc: sc.opacities),
           "cov3D_precomp": stack(lambda sc: cov6(sc.covariances)), "scales": stack(lambda sc: sc.scales),
           "rotations": stack(lambda sc: sc.rotations)}
    if use_sh:
        ins["shs"] = stack(lambda sc: sc.harmonics.permute(0, 2, 1))
    return cams, ins
