"""Strict gradient parity: the element-wise 1e-3 rule on every Gaussian, with the oracle's fragile pixels taken out of the
cotangent instead of exempting the Gaussians behind them.

A pixel's share of every gradient is proportional to the cotangent at that pixel (dL/dcolour, dL/ddepth, dL/dalpha): each
term of the backward's per-pixel sum is a product with it.  So where the cotangent is zero at the pixels on which the oracle
saw a discontinuous decision close to its threshold (alpha >= 1/255, T < 1e-4, near-equal depths: `px_fragile`), a
decision that a kernel takes the other way round there cannot reach any gradient, and no Gaussian needs a looser bound.
What is left are the decisions that belong to a Gaussian rather than to a pixel: its radius or near-plane cull (`geom_fragile`),
the anti-aliasing clamp of its opacity compensation (`near_clamp`), and an SH colour whose value before the clamp at 0 is
within rounding of zero.  Only those Gaussians stay exempt, and there must be few of them.

tests/util.py's `check_grad` (the full cotangent, looser bounds for Gaussians that touch a fragile pixel) stays as it is;
the tests that use these helpers are tests/test_strict_parity_cpu.py and tests/test_gpu_strict_gradients.py."""
from __future__ import annotations

import numpy as np
import torch

from tests.sh4_oracle import sh_basis
from tests.util import GRAD_RTOL

# SH colours within this band (relative to the sum of the magnitudes of their terms, plus the 0.5 offset) of the clamp at
# 0 are undecided: fp32 evaluates that sum to a few 1e-7 of it, and the clamp switches the colour's gradient on or off.
SH_CLAMP_BAND = 1e-5
# at most this many per-Gaussian decisions (per Gaussian, + 2) may be exempt from the strict rule
MAX_EXEMPT_FRAC = 1e-3
# share of the Gaussians that reach the image under the full cotangent that must keep a non-zero masked gradient
MIN_LIVE_FRAC = 0.9


def _np64(a):
    return a.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(a) else np.asarray(a, np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# fragile pixels and the masked cotangent
# ---------------------------------------------------------------------------------------------------------------------
def fragile_pixels(orc) -> np.ndarray:
    """Union of the fragile-pixel masks of every render inside an oracle: bool [H,W] for an OracleRender, [V,H,W] for the
    batched oracles (OracleBatch, ShOracleBatch, AAOracle, AlphaOracle, DepthModeOracle)."""
    if hasattr(orc, "ob_alpha"):                        # AlphaOracle: the alpha render and its base
        return orc.frag | fragile_pixels(orc.base)
    if hasattr(orc, "ob_depth"):                        # DepthModeOracle: the depth render and the colour render
        return orc.frag | orc.frag_color
    if hasattr(orc, "near_clamp"):                      # AAOracle: the per-view oracles, plus the clamp's footprint
        return orc.frag | np.concatenate([fragile_pixels(o) for o in orc.views])
    if hasattr(orc, "batch"):                           # ShOracleBatch
        return fragile_pixels(orc.batch)
    if hasattr(orc, "views"):                           # OracleBatch
        return np.stack([r.px_fragile for r in orc.views])
    return orc.px_fragile


def masked_cotangent(dL, frag) -> np.ndarray:
    """dL [V,3,H,W] / [3,H,W] (colour) or [V,H,W] / [H,W] (depth, alpha) with zeros at the fragile pixels frag [V,H,W] /
    [H,W]; same dtype as dL."""
    dL = np.asarray(dL)
    frag = np.asarray(frag, bool)
    if dL.ndim == frag.ndim + 1:
        frag = np.expand_dims(frag, -3)
    assert dL.ndim == frag.ndim, (dL.shape, frag.shape)
    return np.where(frag, 0, dL).astype(dL.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# per-Gaussian decisions
# ---------------------------------------------------------------------------------------------------------------------
def sh_near_clamp(means, shs, campos, deg: int, band: float = SH_CLAMP_BAND) -> np.ndarray:
    """bool[P]: Gaussians with a colour channel whose SH value before the clamp at 0, recomputed in fp64, lies within
    `band` (relative to the magnitude of its terms) of zero.  means [P,3] as the renderer saw them, shs [P,M,3]."""
    d = np.asarray(means, np.float64) - np.asarray(campos, np.float64).reshape(1, 3)
    u = d / np.linalg.norm(d, axis=-1, keepdims=True)
    K = (deg + 1) ** 2
    terms = sh_basis(u, deg)[:, :, None] * np.asarray(shs, np.float64)[:, :K, :]      # [P,K,3]
    raw = terms.sum(axis=1) + 0.5
    scale = np.abs(terms).sum(axis=1) + 0.5
    return (np.abs(raw) <= band * scale).any(axis=-1)


def _render_decisions(r) -> np.ndarray:
    # geom_fragile bits (gs_oracle.c): 1 the ceil of the radius, 2 the near-plane cull, 4 the tile rect.  A rect that a
    # kernel may draw one tile wider or narrower needs no exemption: the oracle marks fragile every pixel of such a tile
    # that the Gaussian reaches (alpha >= 1/255), and those pixels are out of the cotangent.
    out = (r.geom_fragile_bits & 3) != 0
    if r.shs is not None and len(out):
        out |= sh_near_clamp(r.means3D, r.shs, r.campos, r.sh_eval_degree)
    return out


def _per_scene(view_masks, S: int, VPS: int) -> np.ndarray:
    P = view_masks[0].shape[-1]
    out = np.zeros((S, P), bool)
    for v, m in enumerate(view_masks):
        out[v // VPS] |= np.asarray(m).reshape(P)
    return out


def per_gaussian_decisions(orc) -> np.ndarray:
    """The decisions that belong to a Gaussian, not to a pixel: bool [P] for an OracleRender, [S,P] for the batched
    oracles.  A Gaussian is flagged if, in any view, the ceil of its radius or its near-plane cull is undecided
    (`geom_fragile` bits 1 and 2), its SH colour sits at the clamp (`sh_near_clamp`) or its anti-aliasing ratio sits at
    the clamp (AAOracle.near_clamp)."""
    if hasattr(orc, "ob_alpha"):
        return per_gaussian_decisions(orc.base) | per_gaussian_decisions(orc.ob_alpha)
    if hasattr(orc, "ob_depth"):
        return per_gaussian_decisions(orc.ob_color) | per_gaussian_decisions(orc.ob_depth)
    if hasattr(orc, "near_clamp"):
        views = [per_gaussian_decisions(o)[0] | orc.near_clamp[v] for v, o in enumerate(orc.views)]
        return _per_scene(views, orc.S, orc.VPS)
    if hasattr(orc, "batch"):                           # ShOracleBatch: the colours are its own, evaluated to band 4
        out = per_gaussian_decisions(orc.batch)
        for v in range(orc.V):                          # dirs: unit vectors from the camera, so campos is the origin
            out[v // orc.VPS] |= sh_near_clamp(orc.dirs[v], orc.shs[v // orc.VPS], np.zeros(3), orc.deg)
        return out
    if hasattr(orc, "views"):
        return _per_scene([_render_decisions(r) for r in orc.views], orc.S, orc.VPS)
    return _render_decisions(orc)


def check_exempt(label, exempt) -> int:
    """Per-Gaussian decisions must stay rare: at most 1e-3 of the Gaussians + 2 (per scene when exempt is [S,P])."""
    ex = np.asarray(exempt, bool)
    ex = ex.reshape(-1, ex.shape[-1])
    n = int(ex.sum())
    P = ex.shape[-1]
    print(f"[strict] {label}: per-Gaussian decisions exempt {n} of {ex.size} "
          f"(per scene {ex.sum(axis=1).tolist()}, bound {MAX_EXEMPT_FRAC * P + 2:.0f})")
    assert (ex.sum(axis=1) <= MAX_EXEMPT_FRAC * P + 2).all(), (label, ex.sum(axis=1))
    return n


# ---------------------------------------------------------------------------------------------------------------------
# the strict criterion
# ---------------------------------------------------------------------------------------------------------------------
def strict_report(name, ours, ref, exempt=None, bands=None) -> dict:
    """|a - b| <= 1e-3 (|b| + rms(b)) element-wise, per tensor and per SH band (rms per band, over every Gaussian), for
    every Gaussian outside `exempt`.  ours, ref: [N, ...]; exempt: bool[N] or None."""
    a = _np64(ours)
    b = _np64(ref).reshape(a.shape)
    N = a.shape[0]
    ex = np.zeros(N, bool) if exempt is None else np.asarray(exempt, bool).reshape(N)
    keep = ~ex
    rep = {"name": name, "elements": int(a[keep].size), "exempt_gaussians": int(ex.sum()), "worst_ratio": 0.0,
           "worst_at": None, "gaussians_over_tol": 0}
    over = np.zeros(N, bool)
    for label, sl in ([("all", slice(None))] if bands is None else bands):
        aa, bb = (a, b) if bands is None else (a[:, sl], b[:, sl])
        if aa.size == 0:
            continue
        rms = float(np.sqrt(np.mean(bb * bb)))
        ratio = (np.abs(aa - bb) / (np.abs(bb) + rms + 1e-300)).reshape(N, -1)
        ratio[ex] = 0.0
        over |= ratio.max(axis=1) > GRAD_RTOL
        i, j = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        if ratio[i, j] > rep["worst_ratio"]:
            rep.update(worst_ratio=float(ratio[i, j]), worst_at=(int(i), label, int(j)),
                       worst_ours=float(aa.reshape(N, -1)[i, j]), worst_ref=float(bb.reshape(N, -1)[i, j]), worst_rms=rms)
    rep["gaussians_over_tol"] = int(over.sum())
    return rep


def check_grad_strict(name, ours, ref, exempt=None, bands=None) -> dict:
    rep = strict_report(name, ours, ref, exempt, bands)
    print(f"[strict] grad {rep}")
    assert rep["gaussians_over_tol"] == 0, rep
    return rep


# ---------------------------------------------------------------------------------------------------------------------
# the masked run still tests its regime
# ---------------------------------------------------------------------------------------------------------------------
def _reach(g) -> np.ndarray:
    """Per Gaussian (per scene and Gaussian for batched gradients): |dL/dopacity| + |dL/dmeans3D|."""
    o = np.abs(_np64(g["opacities"])).reshape(-1)
    return o + np.abs(_np64(g["means3D"])).reshape(o.size, -1).sum(axis=1)


def early_terminated(orc) -> np.ndarray:
    """bool [H,W] / [V,H,W]: pixels whose walk stopped because the next Gaussian that reaches them would take T below
    1e-4 (tests/test_gpu_regimes.py's `_termination`)."""
    from tests.test_gpu_regimes import _termination
    if hasattr(orc, "views"):
        return np.stack([early_terminated(r) for r in orc.views])
    return _termination(orc)[0]


def check_masked_regime(label, frag, max_fragile, g_masked, g_full, early=None) -> dict:
    """The masked cotangent leaves the regime under test: the masked pixel fraction stays within the regime's own
    `max_fragile`; at least 90 % of the Gaussians that reach the image (a non-zero gradient under the full cotangent) keep
    a non-zero gradient; and, where `early` (early-terminated pixels) is given, some unmasked pixels still stop early."""
    frag = np.asarray(frag, bool)
    full, masked = _reach(g_full) > 0, _reach(g_masked) > 0
    rep = {"masked_pixel_frac": float(frag.mean()), "max_fragile": max_fragile, "reach_image": int(full.sum()),
           "live_frac": float(masked[full].mean()) if full.any() else 0.0}
    if early is not None:
        rep["early_unmasked_pixels"] = int((np.asarray(early, bool) & ~frag).sum())
    print(f"[strict] {label}: {rep}")
    assert rep["masked_pixel_frac"] <= max_fragile, (label, rep)
    assert full.any() and rep["live_frac"] >= MIN_LIVE_FRAC, (label, rep)
    if early is not None:
        assert rep["early_unmasked_pixels"] > 0, (label, rep)
    return rep
