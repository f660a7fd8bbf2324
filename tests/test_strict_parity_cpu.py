"""The strict gradient rule of tests/strict_parity.py, pinned on the CPU with the fp32 C oracle standing in for a kernel and
the fp64 C oracle as the reference:
  * with masked cotangents the fp32 oracle meets the strict 1e-3 rule on every Gaussian, with no exemption, on the scenes
    the GPU suite's gradient tests are built on -- with a recorded margin (worst ratio <= 3e-4);
  * masking is exact: the gradient under the full cotangent is the masked one plus the one of the fragile pixels alone;
  * the loose rule's blind spot is real: a 0.5 % error on every affected Gaussian, or one dropped per-pixel term, passes
    tests/util.py's check_grad and fails check_grad_strict."""
import numpy as np
import pytest

from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.strict_parity import (check_exempt, check_grad_strict, check_masked_regime, fragile_pixels, masked_cotangent,
                                 per_gaussian_decisions, strict_report)
from tests.util import SH_BANDS, affected_gaussians, check_grad, oracle_view

STRICT_MARGIN = 3e-4
SCENES = {
    "4000 Gaussians, 48x64": lambda: make_scene(4000, 2, 48, 64, seed=3),
    "20000 Gaussians, 70x50": lambda: make_scene(20000, 3, 70, 50, seed=5),
    "pixel-aligned 64x64": lambda: make_pixel_aligned_scene(64, 64, 3, seed=0),
}
NAMES = ("means3D", "means2D", "opacities", "shs", "cov3D_precomp")


def _bands(name):
    return SH_BANDS if name == "shs" else None


def _incoming(orc64, v, seed):
    """MSE against a seeded target (from the fp64 image) and a seeded depth field: the same fp32 arrays for both oracles."""
    H, W = orc64.H, orc64.W
    target = make_target(1, H, W, seed=seed + v)[0].numpy()
    dL = (2 * (orc64.color - target) / target.size).astype(np.float32)
    dLd = (np.random.default_rng(seed + v).standard_normal((H, W)) * 1e-3 / (H * W)).astype(np.float32)
    return dL, dLd


def _pair(sc, v):
    return (oracle_view(sc, v, dtype=np.float32, with_depth=True), oracle_view(sc, v, dtype=np.float64, with_depth=True))


@pytest.mark.parametrize("scene", list(SCENES))
def test_fp32_oracle_meets_the_strict_rule_under_masked_cotangents(scene):
    sc = SCENES[scene]()
    P, V = sc.means.shape[0], sc.extrinsics.shape[0]
    worst, affected = {}, np.zeros(P, bool)
    frag_frac = []
    for v in range(V):
        o32, o64 = _pair(sc, v)
        frag = fragile_pixels(o64)
        frag_frac.append(float(frag.mean()))
        affected |= affected_gaussians(o64, frag) | o64.geom_fragile
        check_exempt(f"{scene} view {v}", per_gaussian_decisions(o64))
        dL, dLd = _incoming(o64, v, seed=11)
        dLm, dLdm = masked_cotangent(dL, frag), masked_cotangent(dLd, frag)
        g32, g64 = o32.backward(dLm, dLdm), o64.backward(dLm, dLdm)
        check_masked_regime(f"{scene} view {v}", frag, 0.03, g64, o64.backward(dL, dLd))
        for name in NAMES:
            rep = check_grad_strict(f"{scene} view {v} fp32 vs fp64 dL/d{name}", g32[name], g64[name], None,
                                    _bands(name))
            worst[name] = max(worst.get(name, 0.0), rep["worst_ratio"])
    print(f"[strict] {scene}: fragile pixels {np.mean(frag_frac):.2%}, affected Gaussians {affected.mean():.1%}, "
          f"masked worst ratio per tensor (no exemption) {worst}")
    assert max(worst.values()) <= STRICT_MARGIN, worst


def test_masking_is_exact_in_the_fp64_oracle():
    """Gradients are linear in the cotangent: full = masked + fragile-only, to rounding of fp64."""
    sc = SCENES["pixel-aligned 64x64"]()
    for v in range(2):
        o64 = oracle_view(sc, v, dtype=np.float64, with_depth=True)
        frag = fragile_pixels(o64)
        assert frag.any()
        dL, dLd = (a.astype(np.float64) for a in _incoming(o64, v, seed=12))
        dLm, dLdm = masked_cotangent(dL, frag), masked_cotangent(dLd, frag)
        full, masked, rest = o64.backward(dL, dLd), o64.backward(dLm, dLdm), o64.backward(dL - dLm, dLd - dLdm)
        for name in NAMES:
            err = np.abs(full[name] - (masked[name] + rest[name])).max() / np.abs(full[name]).max()
            print(f"[strict] masking view {v} dL/d{name}: |full - (masked + fragile-only)| / max|full| = {err:.1e}")
            assert err <= 1e-12, (name, err)


def _verdicts(label, loose, strict):
    print(f"[strict] mutation {label}: loose check {'accepts' if loose else 'rejects'}, strict check "
          f"{'accepts' if strict else 'rejects'}")
    assert loose and not strict, label


def _loose_accepts(name, ours, ref, aff):
    try:
        check_grad(name, ours, ref, aff, _bands(name.split("/d")[-1]))
        return True
    except AssertionError:
        return False


def test_mutations_the_loose_rule_accepts_and_the_strict_rule_rejects():
    sc = SCENES["4000 Gaussians, 48x64"]()
    v = 1
    o32, o64 = _pair(sc, v)
    frag = fragile_pixels(o64)
    aff = affected_gaussians(o64, frag) | o64.geom_fragile
    dL, dLd = _incoming(o64, v, seed=13)
    dLm, dLdm = masked_cotangent(dL, frag), masked_cotangent(dLd, frag)
    full32, full64 = o32.backward(dL, dLd), o64.backward(dL, dLd)
    masked32, masked64 = o32.backward(dLm, dLdm), o64.backward(dLm, dLdm)
    print(f"[strict] mutations on view {v}: {aff.sum()} of {o64.P} Gaussians affected")

    # 1. every affected Gaussian's gradient 0.5 % off
    scale = np.where(aff, 1 + 5e-3, 1.0)
    for name in ("means3D", "opacities", "shs", "cov3D_precomp"):
        s = scale.reshape((-1,) + (1,) * (full32[name].ndim - 1))
        loose = _loose_accepts(f"x1.005 dL/d{name}", full32[name] * s, full64[name], aff)
        strict = strict_report(f"x1.005 dL/d{name}", masked32[name] * s, masked64[name], None,
                               _bands(name))["gaussians_over_tol"] == 0
        _verdicts(f"affected x(1 + 5e-3), dL/d{name}", loose, strict)

    # 2. one term dropped: an affected Gaussian loses the share of one non-fragile pixel (2e-3 .. 8e-3 of its gradient)
    g = np.abs(full64["opacities"][:, 0])
    rms = np.sqrt(np.mean(full64["opacities"] ** 2))
    cand = np.nonzero(aff & (g > 3 * rms))[0]
    cand = cand[np.argsort(-g[cand])][:20]
    xy = o64.xy
    H, W = o64.H, o64.W
    found = None
    for i in cand:
        cx, cy = int(round(xy[i, 0])), int(round(xy[i, 1]))
        r = int(o64.radii[i])
        for y in range(max(0, cy - r), min(H, cy + r + 1)):
            for x in range(max(0, cx - r), min(W, cx + r + 1)):
                if frag[y, x]:
                    continue
                one, oned = np.zeros_like(dL), np.zeros_like(dLd)
                one[:, y, x], oned[y, x] = dL[:, y, x], dLd[y, x]
                term = o64.backward(one, oned)["opacities"][i, 0]
                if 2e-3 <= abs(term) / g[i] <= 8e-3:
                    found = (int(i), y, x, float(term))
                    break
            if found:
                break
        if found:
            break
    assert found is not None, "no (Gaussian, pixel) pair with a 2e-3 .. 8e-3 share"
    i, y, x, term = found
    print(f"[strict] dropped term: Gaussian {i}, pixel (y={y}, x={x}), term {term:.3e} = {abs(term) / g[i]:.2e} of "
          f"dL/dopacity {full64['opacities'][i, 0]:.3e}")
    loose_in, strict_in = full32["opacities"].copy(), masked32["opacities"].copy()
    loose_in[i, 0] -= term
    strict_in[i, 0] -= term
    loose = _loose_accepts("dropped term dL/dopacities", loose_in, full64["opacities"], aff)
    strict = strict_report("dropped term dL/dopacities", strict_in, masked64["opacities"])["gaussians_over_tol"] == 0
    _verdicts("one per-pixel term dropped, dL/dopacities", loose, strict)
