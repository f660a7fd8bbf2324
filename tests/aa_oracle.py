"""Anti-aliased rasterization (GS_FLAG_ANTIALIAS) from the fp64 oracles, by composition.

The rasterizer's oracles (oracle/gs_oracle.c, oracle/torch_oracle.py) draw each splat at its own opacity.  Anti-aliasing
changes one thing: view v draws Gaussian i at o_i * rho_vi, rho = sqrt(max(2.5e-5, det0 / det1)), det0 = a0 c0 - b^2 of
the projected 2-D covariance (a0, b, c0) before the dilation h and det1 = (a0 + h)(c0 + h) - b^2 after it.  Conic, radius
and tiles stay those of the dilated covariance, which the oracles already draw.  So:
  * rho_v is computed here in fp64 from a differentiable restatement of the projected covariance (the one of
    oracle/torch_oracle.py: view-scaled mean and covariance, guard-band-clamped Jacobian);
  * forward: view v is the oracle's render of that view alone at opacities o * rho_v (any per-view oracle: the batched C
    oracle by default, or tests.alpha_oracle.AlphaOracle, tests.sh4_oracle.ShOracleBatch,
    tests.depth_modes_oracle.DepthModeOracle built for the one view);
  * backward: each view's oracle returns dL/do'_v among its gradients; dL/do = sum_v rho_v dL/do'_v, and
    sum_v o dL/do'_v rho_v is differentiated by autograd into means, covariances or scales / rotations.
tests/test_antialias_cpu.py pins the composition to an autograd restatement and to finite differences, and rho to the
dilated covariance the C oracle's own conic implies."""
from __future__ import annotations

import numpy as np
import torch

from tests.batch_oracle import _np, batch_view_settings, oracle_batch

RATIO_MIN = 2.5e-5
SCENE_KEYS = ("means3D", "shs", "scales", "rotations", "cov3D_precomp")
VIEW_KEYS = ("means2D", "colors_precomp")


def sigma3(ins: dict, k: int, scale_modifier: float = 1.0) -> torch.Tensor:
    """(P,3,3) world covariance of scene k from cov3D_precomp [S,P,6] or scales [S,P,3] + rotations [S,P,4] (torch)."""
    if ins.get("cov3D_precomp") is not None:
        c = ins["cov3D_precomp"][k]
        P = c.shape[0]
        return torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], -1).reshape(P, 3, 3)
    r, x, y, z = ins["rotations"][k].unbind(-1)
    P = r.shape[0]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(P, 3, 3)
    sv = scale_modifier * ins["scales"][k]
    return R @ torch.diag_embed(sv * sv) @ R.transpose(-1, -2)


def cov2d(st, means, Sigma):
    """(a0, b, c0): the projected 2-D covariance BEFORE the dilation of view settings `st` (OracleSettings) for view-scaled
    means (P,3) and covariances (P,3,3); fp64 torch, differentiable, as oracle/torch_oracle.py projects it."""
    dt = means.dtype
    view = torch.as_tensor(np.asarray(st.viewmatrix, np.float64), dtype=dt).reshape(4, 4)
    P = means.shape[0]
    p_view = torch.cat([means, torch.ones(P, 1, dtype=dt)], -1) @ view
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


def aa_ratio(a0, b, c0, h):
    return (a0 * c0 - b * b) / ((a0 + h) * (c0 + h) - b * b)


def aa_rho(ratio):
    """rho = sqrt(max(RATIO_MIN, ratio)); below the clamp a constant (zero gradient), as the kernels differentiate it."""
    if torch.is_tensor(ratio):
        return torch.sqrt(torch.where(ratio > RATIO_MIN, ratio, torch.full_like(ratio, RATIO_MIN)))
    return np.sqrt(np.maximum(RATIO_MIN, ratio))


def _slice_settings(bs, v: int):
    """BatchSettings of view v alone."""
    one = lambda t: None if t is None else t[v:v + 1]
    return bs._replace(viewmatrix=one(bs.viewmatrix), projmatrix=one(bs.projmatrix), campos=one(bs.campos), bg=one(bs.bg),
                       tanfov=one(bs.tanfov), view_scale=one(bs.view_scale),
                       depth_near_far=one(getattr(bs, "depth_near_far", None)))


def _render_of(o):
    """The OracleRender inside a one-view oracle (for the fragile-pixel footprint)."""
    for attr in ("views", "batch", "base", "ob_color"):
        x = getattr(o, attr, None)
        if x is not None:
            return x[0] if isinstance(x, list) else _render_of(x)
    return o


def _default_view_oracle(bs_v, ins_v):
    return oracle_batch(bs_v, dtype=np.float64, **ins_v)


class AAOracle:
    """bs: BatchSettings with CPU tensors; ins: the Gaussian inputs of rasterize_batch.  `view_oracle(bs_v, ins_v)` builds
    the oracle of one view (a one-view BatchSettings and inputs with S = 1 and the compensated opacities); its attributes
    are stacked over the views by `stack(name)`.  `rho`, `ratio` [V,P]; `frag` [V,H,W]: pixels a splat whose ratio lies
    within `clamp_band` (relative) of the clamp can reach -- rho's derivative jumps there."""

    def __init__(self, bs, ins, view_oracle=None, clamp_band=1e-3):
        V = int(bs.viewmatrix.shape[0])
        self.ins = {k: (None if v is None else torch.as_tensor(_np(v, np.float64))) for k, v in ins.items()}
        S, P = self.ins["means3D"].shape[:2]
        self.S, self.P, self.V, self.VPS = S, P, V, V // S
        self.M = 0 if self.ins.get("shs") is None else self.ins["shs"].shape[2]
        vs = np.ones(V) if bs.view_scale is None else _np(bs.view_scale, np.float64).reshape(V)
        self.s = vs.astype(np.float32).astype(np.float64)   # the kernels hold s in fp32
        self.bs = bs
        self.settings = [batch_view_settings(bs, v, self.M) for v in range(V)]
        with torch.no_grad():
            self.ratio = self._ratio(self.ins).numpy()
        self.rho = aa_rho(self.ratio)
        self.opac = self.ins["opacities"].reshape(S, P).numpy()
        self.near_clamp = np.abs(self.ratio / RATIO_MIN - 1.0) < clamp_band
        mk = view_oracle or _default_view_oracle
        self.views = []
        for v in range(V):
            k = v // self.VPS
            ins_v = {}
            for name, t in self.ins.items():
                if t is None:
                    continue
                ins_v[name] = t[v:v + 1] if name == "colors_precomp" else t[k:k + 1]
            ins_v["opacities"] = torch.as_tensor(self.opac[k] * self.rho[v])[None]
            self.views.append(mk(_slice_settings(bs, v), ins_v))
        self.frag = np.stack([self._footprint(v) for v in range(V)])

    def _ratio(self, ins) -> torch.Tensor:
        out = []
        for v in range(self.V):
            k, s = v // self.VPS, float(self.s[v])
            st = self.settings[v]
            Sig = sigma3(ins, k, float(self.bs.scale_modifier)) * (s * s)
            a0, b, c0 = cov2d(st, ins["means3D"][k] * s, Sig)
            out.append(aa_ratio(a0, b, c0, st.dilation))
        return torch.stack(out)

    def _footprint(self, v) -> np.ndarray:
        r = _render_of(self.views[v])
        H, W = r.H, r.W
        ids = np.nonzero(self.near_clamp[v] & (r.radii > 0))[0]
        out = np.zeros((H, W), bool)
        if len(ids) == 0:
            return out
        xy, co = r.xy.astype(np.float64)[ids], r.conic_opacity.astype(np.float64)[ids]
        yy, xx = np.mgrid[0:H, 0:W]
        for i in range(len(ids)):
            dx, dy = xy[i, 0] - xx, xy[i, 1] - yy
            power = -0.5 * (co[i, 0] * dx * dx + co[i, 2] * dy * dy) - co[i, 1] * dx * dy
            out |= (power <= 1e-6) & (co[i, 3] * np.exp(np.minimum(power, 0.0)) >= (1 / 255) * 0.99)
        return out

    def stack(self, name):
        vals = [getattr(o, name) for o in self.views]
        return None if vals[0] is None else np.concatenate([np.asarray(x) for x in vals])

    @property
    def color(self):
        return self.stack("color")

    @property
    def depth(self):
        return self.stack("depth")

    @property
    def radii(self):
        return self.stack("radii")

    def affected(self) -> np.ndarray:
        out = np.zeros((self.S, self.P), bool)
        for v, o in enumerate(self.views):
            out[v // self.VPS] |= o.affected()[0] | self.near_clamp[v]
        return out

    def check_conic(self) -> float:
        """Largest relative difference between the dilated covariance (a0 + h, b, c0 + h) of the restatement and the one the
        C oracle's conic implies, over the visible (view, Gaussian) pairs; and the oracle's opacity must be o * rho."""
        worst = 0.0
        with torch.no_grad():
            for v in range(self.V):
                k, s = v // self.VPS, float(self.s[v])
                st = self.settings[v]
                a0, b, c0 = (t.numpy() for t in cov2d(st, self.ins["means3D"][k] * s,
                                                      sigma3(self.ins, k, float(self.bs.scale_modifier)) * (s * s)))
                r = _render_of(self.views[v])
                vis = r.radii > 0
                co = r.conic_opacity.astype(np.float64)[vis]
                det = co[:, 0] * co[:, 2] - co[:, 1] ** 2
                dil = np.stack([co[:, 2] / det, -co[:, 1] / det, co[:, 0] / det], -1)
                want = np.stack([a0 + st.dilation, b, c0 + st.dilation], -1)[vis]
                scale = np.abs(want).max(axis=1, keepdims=True)
                worst = max(worst, float((np.abs(dil - want) / scale).max()) if vis.any() else 0.0)
                np.testing.assert_allclose(co[:, 3], (self.opac[k] * self.rho[v])[vis], rtol=1e-12, atol=0)
        return worst

    def backward(self, *args) -> dict:
        """args: the per-view oracle's backward arguments, each [V,...] (or None).  Returns the gradients rasterize_batch
        returns, per scene where the input is per scene."""
        S, P, V = self.S, self.P, self.V
        g: dict = {}
        dlo = np.zeros((V, P))
        extra: dict = {}
        for v, o in enumerate(self.views):
            k = v // self.VPS
            gv = o.backward(*[None if a is None else np.asarray(_np(a))[v:v + 1] for a in args])
            dlo[v] = np.asarray(gv["opacities"]).reshape(P)
            for name, x in gv.items():
                if name == "opacities":
                    continue
                if x is None:
                    g.setdefault(name, None)
                    continue
                x = np.asarray(x, np.float64)
                if name in SCENE_KEYS:
                    if g.get(name) is None:
                        g[name] = np.zeros((S,) + x.shape[1:])
                    g[name][k] += x[0]
                else:
                    extra.setdefault(name, []).append(x)
        for name, xs in extra.items():
            g[name] = np.concatenate(xs) if xs[0].ndim and xs[0].shape[0] == 1 else np.stack(xs)
        g["opacities"] = np.zeros((S, P))
        for v in range(V):
            g["opacities"][v // self.VPS] += self.rho[v] * dlo[v]
        # the rho chain: d/dx of sum_v o dL/do'_v rho_v(x)
        leaves = {k: (t.clone().requires_grad_(True) if t is not None and k in ("means3D", "scales", "rotations",
                                                                               "cov3D_precomp") else t)
                  for k, t in self.ins.items()}
        w = torch.as_tensor(np.stack([self.opac[v // self.VPS] * dlo[v] for v in range(V)]))
        (aa_rho(self._ratio(leaves)) * w).sum().backward()
        for k in ("means3D", "scales", "rotations", "cov3D_precomp"):
            t = leaves.get(k)
            if t is not None and t.grad is not None:
                g[k] = g[k] + t.grad.numpy()
        return g
