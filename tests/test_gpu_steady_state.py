"""The steady state of lazy depth strata (DESIGN.md 5.2), held to the fp64 oracles under every output, backward and feature.

From the third call of a shape on, k_stratum_rank_sort sorts only the strata each tile's previous forward read, and
k_composite_fwd<..., LAZY=true> sorts any further stratum it reaches, appends it to point_list and extends ranges[vt].y;
every backward (atomic, deterministic, camera) reads those lists.  Every case drives one shape through

    1 dense: exact     2 dense: trial (table reset to "all")     3, 4 dense: lazy, the table learned: strata skipped
    5 dense, moved by about a pixel: lazy     6 faint (opacities / 20): every skipped stratum sorted by the compositor
    7 dense: the table learned back

(tests/test_steady_state_policy_cpu.py replays the same sequences through the binning policy) and checks
  (a) colour, radii, depth, alpha, and the deterministic backward's gradients (cameras included) bit for bit against the
      same sequence under GS_TUNE_ALL_STRATA (every stratum sorted up front), each setting on a stream -- a context and a
      "strata needed" table -- of its own;
  (b) the default (atomic) backward against ALL_STRATA's and against the deterministic one of the same call:
      max |a - b| <= 2e-5 max |b|;
  (c) calls 4 and 6 against the fp64 oracle of the feature (tests/util.py's image and gradient rules).
Saturation is measured on a side stream (GS_TUNE_NO_SPECULATION, alpha requested): where the compositor stops, T_final
lies in [1e-4, 1e-2) -- the stopping splat is not added and alpha is clamped at 0.99 -- so a pixel counts as saturated at
alpha >= 0.99.  Each test's shape (Gaussians per scene) is one no other test renders; the module starts and ends with no
context cached."""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import Scene, make_scene
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.regimes import TANFOV, _U, _at_pixels, _with_extra
from tests.test_gpu_forward_variants import _with_culled
from tests.test_gpu_regimes import _settings
from tests.util import FRAGILE_RGB_TOL, RGB_TOL, SH_BANDS, check_grad, grad_report

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ALL = _capi.GS_TUNE_ALL_STRATA
HW = (64, 96)                    # 4 x 6 tiles per view
DENSE = 46_000                   # 7.5 Gaussians per pixel, as C2 (500k over 256 x 256): saturates
ATOMIC_RTOL = 2e-5               # test_gpu_parity.py's criterion for backward variants
SAT = 0.99


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    """Contexts are cached per (device, stream) and torch reuses streams: start and end with none cached."""
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    torch.use_deterministic_algorithms(False)
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()


# ---------------------------------------------------------------------------------------------------------------------
# the engine: one call, a sequence under the default and under ALL_STRATA, the comparisons
# ---------------------------------------------------------------------------------------------------------------------
class Call(NamedTuple):
    bs: object                      # BatchSettings with device cameras
    ins: dict                       # device inputs
    backward: bool = True
    means2D: bool = False
    view_grad: bool = False         # the view matrix requires grad (the depth channel's z column)
    cam: bool = False               # viewmatrix, projmatrix, campos require grad, camera_gradients on
    label: str = ""


def _names(bs):
    return ["color", "radii"] + (["depth"] if bs.with_depth else []) + (["alpha"] if bs.with_alpha else [])


def _incoming(bs, seed=5):
    V, H, W = bs.viewmatrix.shape[0], bs.image_height, bs.image_width
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: (torch.randn(*s, generator=g) / (H * W)).to(DEV)
    return {"color": r(V, 3, H, W), "depth": r(V, H, W) if bs.with_depth else None,
            "alpha": r(V, H, W) if bs.with_alpha else None}


def _one(c: Call, tuning: int):
    """Forward of c under `tuning` on the current stream; then the deterministic backward and the atomic one of the same
    saved state.  Returns {"out", "stats", "det", "atomic"}."""
    from pf3plat_b200.rasterizer import last_stats, rasterize_batch
    bs = c.bs._replace(tuning=c.bs.tuning | tuning)
    leaves = {k: v.clone().requires_grad_(c.backward) for k, v in c.ins.items()}
    V, P = bs.viewmatrix.shape[0], c.ins["means3D"].shape[1]
    if c.means2D:
        leaves["means2D"] = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    if c.cam:
        for k in ("viewmatrix", "projmatrix", "campos"):
            leaves[k] = getattr(bs, k).clone().requires_grad_(True)
        bs = bs._replace(viewmatrix=leaves["viewmatrix"], projmatrix=leaves["projmatrix"], campos=leaves["campos"],
                         camera_gradients=True)
    elif c.view_grad:
        leaves["viewmatrix"] = bs.viewmatrix.clone().requires_grad_(True)
        bs = bs._replace(viewmatrix=leaves["viewmatrix"], camera_gradients=False)
    else:
        bs = bs._replace(camera_gradients=False)
    gin = {k: v for k, v in leaves.items() if k not in ("viewmatrix", "projmatrix", "campos")}
    out = dict(zip(_names(bs), rasterize_batch(bs, **gin)))
    res = {"out": {k: v.detach().clone() for k, v in out.items()}, "stats": last_stats(DEV), "det": None, "atomic": None}
    if c.backward:
        inc = _incoming(bs)
        ts = [out[k] for k in ("color", "depth", "alpha") if inc[k] is not None]
        gs = [inc[k] for k in ("color", "depth", "alpha") if inc[k] is not None]
        for det in (True, False):
            for t in leaves.values():
                t.grad = None
            torch.use_deterministic_algorithms(det)
            try:
                torch.autograd.backward(ts, gs, retain_graph=det)
            finally:
                torch.use_deterministic_algorithms(False)
            res["det" if det else "atomic"] = {k: t.grad.clone() for k, t in leaves.items() if t.grad is not None}
    return res


def _sequence(calls, extras=(0, ALL)):
    """The same calls under each tuning in `extras`, each on a stream (a context) of its own."""
    res, streams = {}, []
    for extra in extras:
        s = torch.cuda.Stream(DEV)
        streams.append(s)
        with torch.cuda.stream(s):
            res[extra] = [_one(c, extra) for c in calls]
            s.synchronize()
    return res


def _close(label, a, b):
    scale = float(b.abs().max())
    err = float((a - b).abs().max())
    assert err <= ATOMIC_RTOL * scale, f"{label}: max |diff| {err:.3e} > {ATOMIC_RTOL} x {scale:.3e}"
    return err / scale if scale else 0.0


def _identical(label, res, atomic_calls=(3, 4, 5), ref_key=ALL):
    """(a) and (b).  Returns the default run."""
    lazy, ref = res[0], res[ref_key]
    for i, (r, r0) in enumerate(zip(lazy, ref)):
        for name in r0["out"]:
            a, b = r["out"][name], r0["out"][name]
            assert torch.equal(a, b), f"{label} call {i + 1}: {name} differs (max |diff| " \
                                      f"{float((a.double() - b.double()).abs().max()):.3e})"
        st, st0 = r["stats"], r0["stats"]
        assert st["num_rendered"] == st0["num_rendered"], (label, i + 1, st, st0)
        assert (r["det"] is None) == (r0["det"] is None)
        for k in r0["det"] or {}:
            assert torch.equal(r["det"][k], r0["det"][k]), f"{label} call {i + 1}: deterministic dL/d{k} differs"
        worst = 0.0
        if r["atomic"] is not None and i in atomic_calls:
            for k in r0["atomic"]:
                worst = max(worst, _close(f"{label} call {i + 1}: atomic dL/d{k} vs {ref_key:#x}", r["atomic"][k],
                                          r0["atomic"][k]))
                worst = max(worst, _close(f"{label} call {i + 1}: atomic dL/d{k} vs deterministic", r["atomic"][k],
                                          r["det"][k]))
        print(f"[steady] {label} call {i + 1}: speculative={st['speculative']} D={st['num_rendered']} "
              f"redos={st['overflow_redos']} atomic worst ratio {worst:.2e}")
    return lazy


def _alpha_map(bs, ins):
    """alpha [V,H,W] of an exact render on a stream of its own."""
    from pf3plat_b200.rasterizer import rasterize_batch
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s), torch.no_grad():
        a = rasterize_batch(bs._replace(with_alpha=True, tuning=_capi.GS_TUNE_NO_SPECULATION, camera_gradients=False),
                            **ins)[-1]
        s.synchronize()
    return a


def _saturation(bs, ins):
    """(fraction of pixels at alpha >= SAT, fraction at alpha < 0.999)."""
    a = _alpha_map(bs, ins)
    return float((a >= SAT).float().mean()), float((a < 0.999).float().mean())


# ---------------------------------------------------------------------------------------------------------------------
# oracles
# ---------------------------------------------------------------------------------------------------------------------
def _img(label, got, want, frag, max_frag, tol=RGB_TOL):
    """got, want [V,(C,)H,W]; frag [V,H,W].  The four numbers of SURVEY.md section 7, asserted."""
    g = got.detach().cpu().double().numpy()
    w = np.asarray(want, np.float64)
    err = np.abs(g - w)
    if err.ndim == 4:
        err = err.max(axis=1)
    nf = err[~frag]
    rep = {"pixels": int(err.size), "over_tol": int((err > tol).sum()), "nonfragile_over_tol": int((nf > tol).sum()),
           "fragile_frac": float(frag.mean()), "max_err_nonfragile": float(nf.max()) if nf.size else 0.0,
           "max_err_fragile": float(err[frag].max()) if frag.any() else 0.0}
    print(f"[parity] {label} {rep}")
    assert rep["fragile_frac"] <= max_frag and rep["max_err_nonfragile"] <= tol, (label, rep)
    assert rep["max_err_fragile"] <= max(FRAGILE_RGB_TOL, 50 * tol), (label, rep)


def _check_grad(name, a, b, affected, bands, faint):
    """tests/util.py's rule; in a faint call (opacities 0.0025-0.05) a large share of all splat-pixel pairs sits near the
    alpha >= 1/255 cut, and up to 3e-3 of the affected Gaussians (not 1e-4) may be flipped ones (measured 2.1e-3 on an
    H100).  A flipped Gaussian gains or loses a whole pixel's term, and with few pixels reaching it that term is a large
    share of its gradient: up to 0.5 (measured 0.21).  Unaffected Gaussians keep the strict 1e-3 rule; the bits of every
    call are pinned to ALL_STRATA's regardless."""
    if not faint:
        return check_grad(name, a, b, affected, bands)
    rep = grad_report(name, a, b, affected, bands)
    print(f"[parity] grad (faint) {rep}")
    assert rep["gaussians_over_tol"] == 0, rep
    assert rep["affected_over_1e-2"] <= 3e-3 * rep["affected_gaussians"] + 2, rep
    assert rep["worst_ratio_affected"] <= 0.5, rep
    return rep


def _frag(views, attr="px_fragile"):
    return np.stack([getattr(r, attr) for r in views])


def _cpu(c: Call):
    """The call's settings and inputs on the CPU, for the oracles."""
    d = lambda t: t.cpu() if torch.is_tensor(t) else t
    bs = c.bs._replace(**{k: d(getattr(c.bs, k)) for k in ("viewmatrix", "projmatrix", "campos", "bg", "tanfov",
                                                             "view_scale", "depth_near_far")})
    return bs, {k: v.cpu() for k, v in c.ins.items()}


def _oracle(label, c: Call, r, kind, max_frag=0.08, faint=False):
    """(c): the call's outputs r["out"] and deterministic gradients r["det"] against the fp64 oracle of `kind`."""
    from tests.aa_oracle import AAOracle
    from tests.alpha_oracle import AlphaOracle
    from tests.depth_modes_oracle import DepthModeOracle
    from tests.sh4_oracle import ShOracleBatch
    bs, ins = _cpu(c)
    inc = {k: (None if v is None else v.cpu().double().numpy()) for k, v in _incoming(c.bs).items()}
    dL, w, dA = inc["color"], inc["depth"], inc["alpha"]
    out, got = r["out"], dict(r["det"])
    mode = bs.depth_mode if bs.with_depth else None
    s = bs.view_scale.numpy().astype(np.float32).astype(np.float64)
    wz = None if w is None else (w * s[:, None, None] if mode == "depth" else w)   # "depth" composites s * z

    def base_of(b, i):
        if mode is not None:
            return DepthModeOracle(b, i, mode, b.depth_near_far)
        if kind == "sh4":
            return ShOracleBatch(b, i["means3D"], i["opacities"], i["shs"], deg=4, scales=i.get("scales"),
                                 rotations=i.get("rotations"), cov3D_precomp=i.get("cov3D_precomp"))
        return oracle_batch(b, dtype=np.float64, **i)

    def view_oracle(b, i):
        return AlphaOracle(b, i, base=base_of(b, i)) if b.with_alpha else base_of(b, i)

    orc = AAOracle(bs, ins, view_oracle=view_oracle) if bs.antialiasing else view_oracle(bs, ins)
    args = ([dA] if bs.with_alpha else []) + [dL] + ([wz] if mode is not None else [])
    go = orc.backward(*args)
    aff = orc.affected()
    views = orc.views if bs.antialiasing else [orc]
    aa_frag = orc.frag if bs.antialiasing else False
    bases = [(v.base if bs.with_alpha else v) for v in views]

    def colour_frag(b):
        if mode is not None:
            return b.frag_color
        return _frag((b.batch if kind == "sh4" else b).views)
    cf = np.concatenate([colour_frag(b) for b in bases]) | aa_frag
    _img(f"{label} colour", out["color"], orc.color, cf, max_frag)
    if mode is not None:
        want = np.concatenate([b.depth for b in bases]) * (s[:, None, None] if mode == "depth" else 1.0)
        df = np.concatenate([b.frag for b in bases]) | aa_frag
        _img(f"{label} depth ({mode})", out["depth"], want, df, max_frag, tol=1e-4 * max(float(np.abs(want).max()), 1e-3))
    if bs.with_alpha:
        want = np.concatenate([v.alpha for v in views])
        _img(f"{label} alpha", out["alpha"], want, np.concatenate([v.frag for v in views]) | aa_frag, max_frag)
    S, VPS = aff.shape[0], bs.viewmatrix.shape[0] // aff.shape[0]
    cam = {k: got.pop(k, None) for k in ("viewmatrix", "projmatrix", "campos")}
    for k, g in got.items():
        ref = go[k]
        bands = (SH_BANDS + [("band4", slice(16, 25))] if kind == "sh4" else SH_BANDS) if k == "shs" else None
        if k == "shs" and kind != "sh4":
            g, ref = g[:, :, :16], np.asarray(ref)[:, :, :16]
        per_view = k in ("means2D", "colors_precomp")
        for j in range(g.shape[0]):
            a = aff[j // VPS] if per_view else aff[j]
            _check_grad(f"{label} dL/d{k} {'view' if per_view else 'scene'} {j}", g[j].reshape(g.shape[1], -1),
                        np.asarray(ref[j]).reshape(g.shape[1], -1), a, bands, faint)
    if c.view_grad and cam["viewmatrix"] is not None:
        from tests.chain_oracle import camera_grad_check
        vg = cam["viewmatrix"]
        rest = vg.clone()
        rest[:, :, 2] = 0
        assert int(torch.count_nonzero(rest)) == 0, f"{label}: view-matrix gradient outside the z column"
        camera_grad_check(f"{label} dL/dviewmatrix_z", vg[:, :, 2], go["view_z"], go["view_z_terms"],
                          np.repeat(aff, VPS, axis=0))
    if c.cam:
        from tests.camera_oracle import camera_oracle
        from tests.chain_oracle import camera_grad_check
        ref = camera_oracle(bs, ins, dL, w, dA, antialiasing=bool(bs.antialiasing), depth_mode=mode or "depth",
                            near_far=bs.depth_near_far)
        for name, rr in zip(("viewmatrix", "projmatrix", "campos"), ref):
            V = rr.shape[0]
            camera_grad_check(f"{label} dL/d{name}", cam[name].reshape(V, -1), rr, np.zeros((V, 1) + rr.shape[1:]),
                              np.zeros((V, 1), bool))
    return orc


# ---------------------------------------------------------------------------------------------------------------------
# scenes and the seven-call sequence
# ---------------------------------------------------------------------------------------------------------------------
def _cams(scenes, **kw):
    cams, ins = scene_batch_args(scenes, **kw)
    return {k: v.to(DEV) for k, v in cams.items()}, {k: v.to(DEV) for k, v in ins.items()}


def _near_far(cams):
    near = 1.0 / cams["view_scale"]
    return torch.stack([near, 100 * near], -1)


def _moved(ins, hw, seed):
    """Every mean shifted by about one pixel in the image plane (views differ from view 0 in the image plane only)."""
    g = torch.Generator().manual_seed(seed)
    m = ins["means3D"].cpu()
    px = m[..., 2:3] * (2 * TANFOV / hw[1])
    step = torch.randn(m.shape, generator=g) * px * torch.tensor([1.0, 1.0, 0.0])
    return dict(ins, means3D=(m + step).contiguous().to(DEV))


def _faint(ins):
    return dict(ins, opacities=ins["opacities"] / 20)


def _seven(make_call, ins, hw, seed=3):
    """The sequence of the module docstring; make_call(ins) -> Call."""
    dense = make_call(ins)
    return [dense._replace(backward=False, label="exact"), dense._replace(backward=False, label="trial"),
            dense._replace(label="lazy"), dense._replace(label="lazy, table learned"),
            make_call(_moved(ins, hw, seed))._replace(label="moved"), make_call(_faint(ins))._replace(label="faint"),
            dense._replace(label="dense again")]


def _run_seven(label, calls, kind, oracle_calls=(3, 5), saturates=True, faint=True, max_frag=0.08):
    res = _sequence(calls)
    lazy = _identical(label, res)
    spec = [r["stats"]["speculative"] for r in lazy]
    redos = [r["stats"]["overflow_redos"] for r in lazy]
    print(f"[steady] {label}: speculative per call {spec}, overflow redos {redos}")
    assert spec == [0, 2, 2, 2, 2, 2, 2] and redos[-1] == redos[0], (spec, redos)
    sat = [_saturation(c.bs, c.ins) for c in calls[2:6]]
    print(f"[steady] {label}: saturated fraction calls 3-5 {[round(x[0], 4) for x in sat[:3]]}; faint call 6: "
          f"{sat[3][0]:.4f} saturated, {sat[3][1]:.4f} below alpha 0.999")
    if saturates:   # without it, calls 4 and 5 would skip nothing
        assert min(x[0] for x in sat[:3]) >= 0.9, sat
    if faint:       # and without this, call 6 would sort nothing the table skipped
        assert sat[3][1] >= 0.9, sat
    for i in oracle_calls:
        _oracle(f"{label} call {i + 1} ({calls[i].label})", calls[i], lazy[i], kind, max_frag,
                faint=calls[i].label.startswith("faint"))
    return lazy


# ---------------------------------------------------------------------------------------------------------------------
# 1. every feature in the steady state
# ---------------------------------------------------------------------------------------------------------------------
class Row(NamedTuple):
    label: str
    k: int                                  # culled Gaussians added: the shape no other test renders
    alpha: bool = False
    depth: Optional[str] = None
    aa: bool = False
    sh4: bool = False
    geometry: str = "cov3D"                 # or "scalerot"
    colors: bool = False                    # colors_precomp instead of SH
    means2D: bool = False
    view_grad: bool = False
    cam: bool = False
    scenes: int = 1
    hw: tuple = HW


ROWS = [
    Row("colour only", 101, means2D=True),
    Row("colour + alpha", 102, alpha=True),
    Row("depth z + alpha", 103, alpha=True, depth="depth", view_grad=True),
    Row("disparity", 104, depth="disparity"),
    Row("disparity + alpha", 105, depth="disparity", alpha=True),
    Row("relative disparity", 106, depth="relative_disparity"),
    Row("relative disparity + alpha", 107, depth="relative_disparity", alpha=True),
    Row("log", 108, depth="log"),
    Row("log + alpha", 109, depth="log", alpha=True),
    Row("aa + log + alpha", 110, aa=True, depth="log", alpha=True),
    Row("sh degree 4, scales / rotations", 111, sh4=True, geometry="scalerot"),
    Row("colors_precomp", 112, colors=True, alpha=True),
    # the camera oracle differentiates a dense fp64 render of every tile's whole list: a smaller frame, the same density
    Row("camera gradients, aa + log + alpha", 113, cam=True, aa=True, depth="log", alpha=True, hw=(32, 48)),
    Row("two scenes, ragged view_scale", 114, alpha=True, scenes=2),
]


def _row_call(row: Row, cams, hw):
    def make(ins):
        bs = _settings(cams, hw, sh_degree=4 if row.sh4 else 3, with_depth=row.depth is not None)
        bs = bs._replace(with_alpha=row.alpha, antialiasing=row.aa, sh_eval_max_degree=4 if row.sh4 else 3)
        if row.depth is not None:
            bs = bs._replace(depth_mode=row.depth, depth_near_far=_near_far(cams))
        return Call(bs, ins, means2D=row.means2D, view_grad=row.view_grad, cam=row.cam)
    return make


def _row_inputs(row: Row, hw):
    from tests.sh4_oracle import with_band4
    S = row.scenes
    P = int(7.5 * hw[0] * hw[1]) // S
    scenes = [_with_culled(make_scene(P, 3 if S > 1 else 2, *hw, seed=300 + row.k + j), row.k) for j in range(S)]
    if row.sh4:
        scenes = [with_band4(sc) for sc in scenes]
    near = None
    if S > 1:
        near = 1.0 / np.concatenate([np.linspace(0.8, 1.25, 3), np.linspace(1.1, 0.9, 3)])
    cams, ins = _cams(scenes, near=near)
    keep = ("means3D", "opacities") + (("cov3D_precomp",) if row.geometry == "cov3D" else ("scales", "rotations"))
    out = {k: ins[k] for k in keep}
    if row.colors:
        V = cams["viewmatrix"].shape[0]
        out["colors_precomp"] = torch.rand(V, ins["means3D"].shape[1], 3, generator=torch.Generator().manual_seed(row.k)
                                           ).to(DEV)
    else:
        out["shs"] = ins["shs"]
    return cams, out


@pytest.mark.parametrize("row", ROWS, ids=[r.label for r in ROWS])
def test_feature_in_the_steady_state(row):
    hw = row.hw
    cams, ins = _row_inputs(row, hw)
    calls = _seven(_row_call(row, cams, hw), ins, hw, seed=row.k)
    _run_seven(row.label, calls, "sh4" if row.sh4 else "plain", max_frag=0.12 if row.aa else 0.08)


# ---------------------------------------------------------------------------------------------------------------------
# 2. edge cases of the lazy sort itself
# ---------------------------------------------------------------------------------------------------------------------
def _cloud(sc, n, box, z_lo, z_hi, sig_px, opac, seed, hw):
    """sc plus n splats over the pixel box (u0, v0, u1, v1) of view 0 at depths [z_lo, z_hi), sigma in pixels."""
    g = torch.Generator().manual_seed(seed)
    u0, v0, u1, v1 = box
    z = _U(g, z_lo, z_hi, n)
    means = _at_pixels(_U(g, u0, u1, n), _U(g, v0, v1, n), z, *hw)
    f_px = hw[1] / (2 * TANFOV)
    sigma = _U(g, sig_px[0], sig_px[1], n) * z / f_px
    return _with_extra(sc, means, sigma[:, None] * torch.exp(_U(g, -0.2, 0.2, n, 3)), _U(g, opac[0], opac[1], n), g)


def _plain_call(cams, hw, alpha=True):
    def make(ins):
        bs = _settings(cams, hw, sh_degree=3)._replace(with_alpha=alpha, sh_eval_max_degree=3)
        return Call(bs, ins)
    return make


def _edge(label, sc, k, saturates=True, faint=True, max_frag=0.08, quantise=None):
    hw = sc.image_shape
    cams, ins = _cams([_with_culled(sc, k)])
    ins = {n: ins[n] for n in ("means3D", "opacities", "shs", "cov3D_precomp")}
    calls = _seven(_plain_call(cams, hw), ins, hw, seed=k)
    if quantise is not None:
        # every call's depths on `quantise` levels, so that the boundaries are learned on them too (else the crowded strata
        # overflow); the compositor's CTA-wide rank sort of the faint call must break the ties by index
        for i, c in enumerate(calls):
            m = c.ins["means3D"].clone()
            z = m[..., 2]
            vis = z > 0
            lo, hi = 1.5, 20.0
            zq = lo + torch.round((z - lo) / (hi - lo) * (quantise - 1)) / (quantise - 1) * (hi - lo)
            m[..., 2] = torch.where(vis, zq, z)
            calls[i] = c._replace(ins=dict(c.ins, means3D=m))
        print(f"[regime] {label}: {int(torch.unique(m[..., 2][vis]).numel())} distinct depths")
    return _run_seven(label, calls, "plain", saturates=saturates, faint=faint, max_frag=max_frag), calls


def test_bimodal_depth_with_empty_middle_strata():
    """A faint near layer (depth 2.00-2.02) and an opaque far wall (14-15), nothing between: the per-view octiles fall
    inside the two layers, the strata that straddle the gap hold few or no entries of a tile, and the compositor's
    lazy_sort_next walks from the near layer across them to the wall; the table is learned across them."""
    hw = HW
    sc = make_scene(0, 2, *hw, seed=40)
    box = (-4.0, -4.0, hw[1] + 3.0, hw[0] + 3.0)
    sc = _cloud(sc, 12_000, box, 2.0, 2.02, (0.5, 1.5), (0.01, 0.03), 41, hw)
    sc = _cloud(sc, 30_000, box, 14.0, 15.0, (0.8, 2.0), (0.6, 0.95), 42, hw)
    _edge("bimodal depth", sc, 120, max_frag=0.15)   # the faint layer's splats sit near the 1/255 cut


def test_a_stratum_longer_than_the_compositor_batch():
    """1 100 small splats inside one tile at depths 17.0-17.2: inside the last view octile of the dense background
    (depths 1.5-20, about 4 500 entries per tile list, saturated long before), whose share of that tile's last stratum
    is some 560 more.  The trial's doubled index sub-buckets (about 2 x 1.3 x 5 600 / 8) still hold that stratum and the
    learned capacity stays within the stratum sort's 2 048, so the shape stays on per-view lazy strata: no overflow, no
    per-tile fallback.  In the faint call the compositor sorts that stratum itself: longer than its 256 threads and
    than one 256-entry batch, so each thread ranks several keys and the sorted stratum spans batches.
    (1 500 splats, with their share of the background, would exceed the stratum sort's 2 048 and turn strata off.)

    That the stratum is that long is asserted on the oracle's lists of view 0: the depth range 17.0-17.2 holds under
    1/16 of the view's tile instances, so at most one of the view's octile boundaries (1/8 of its instances apart) falls
    inside it; the clump's tile list holds all 1 100 clump entries, so one of at most two strata holds >= 550."""
    hw = HW
    base = make_scene(DENSE, 2, *hw, seed=43)
    sc = _cloud(base, 1_100, (35.0, 19.0, 44.0, 28.0), 17.0, 17.2, (0.4, 0.8), (0.3, 0.8), 44, hw)
    lazy, calls = _edge("long stratum", sc, 121)
    assert all(r["stats"]["overflow_redos"] == 0 for r in lazy)
    bs, ins = _cpu(calls[3])
    r = oracle_batch(bs, **ins).views[0]
    z = ins["means3D"][0, :, 2].numpy()                         # view 0 is the identity camera: camera z = world z
    pl = np.asarray(r.point_list)
    in_range = int(((z[pl] >= 17.0) & (z[pl] < 17.2)).sum())
    s0, e0 = r.ranges[1 * 6 + 2]                                 # tile (x 2, y 1): pixels 32-47 x 16-31
    ids = np.asarray(pl[s0:e0])
    clump = int(((ids >= DENSE) & (ids < DENSE + 1_100)).sum())
    print(f"[regime] long stratum: view 0 has {len(pl)} tile instances, {in_range} of them at depths 17.0-17.2; "
          f"the clump's tile list is {e0 - s0} long with {clump} clump entries")
    assert in_range * 16 < len(pl) and clump == 1_100


@pytest.mark.parametrize("levels", [8, 64])
def test_depth_ties_in_a_lazily_sorted_stratum(levels):
    # the oracle flags every pixel where two contributors tie in depth as fragile (an order decision at its threshold),
    # so its image check reduces to the fragile bound here; the tie order itself is pinned bit for bit by ALL_STRATA
    _edge(f"{levels} depth levels", make_scene(DENSE, 2, *HW, seed=46), 150 + levels, quantise=levels, max_frag=1.0)


@pytest.mark.parametrize("hw", [(33, 250), (1, 40)], ids=["33x250", "1x40"])
def test_ragged_frames(hw):
    """Edge tiles whose warps lie wholly outside the image (rows 33-47 of the last tile row; rows 1-15 of a 1-pixel frame):
    the reach they record must not cut the next call short.  Both frames saturate in calls 3-5, so the table skips
    strata, and neither does in the faint call, which must sort them again -- the outputs of calls 4-6, bit for bit those
    of ALL_STRATA, are where a wrong reach would show.  The 1-pixel frame's splats are huge (make_scene sizes them by
    1 / h): 150 of them saturate every pixel, and 1/20 of their opacity none."""
    P = int(7.5 * hw[0] * hw[1]) if hw[0] > 1 else 150
    _edge(f"{hw[0]} x {hw[1]}", make_scene(P, 2, *hw, seed=47), 130 + hw[0])


def test_half_dense_half_sparse():
    """The right half saturates, the left never does: need values of 8 next to small ones in one view.  Asserted on the
    alpha of calls 3-5 in columns far from the split (the views are displaced in the image plane)."""
    hw = HW
    sc = make_scene(DENSE, 2, *hw, seed=48)
    keep = (sc.means[:, 0] > 0) | (torch.rand(sc.means.shape[0], generator=torch.Generator().manual_seed(49)) < 0.03)
    kw = {n: getattr(sc, n) for n in ("means", "covariances", "harmonics", "opacities", "scales", "rotations")}
    sc = Scene(sc.extrinsics, sc.intrinsics, sc.near, sc.far, sc.image_shape, sc.background,
               *[kw[n][keep].contiguous() for n in ("means", "covariances", "harmonics", "opacities", "scales", "rotations")])
    _, calls = _edge("half dense, half sparse", sc, 135, saturates=False)
    for c in calls[2:5]:
        a = _alpha_map(c.bs, c.ins)
        left, right = float((a[:, :, :24] < SAT).float().mean()), float((a[:, :, -24:] >= SAT).float().mean())
        print(f"[regime] half dense: {right:.4f} of the right quarter saturated, {left:.4f} of the left quarter not")
        assert left >= 0.9 and right >= 0.9, (left, right)


# ---------------------------------------------------------------------------------------------------------------------
# 3. sequences across calls
# ---------------------------------------------------------------------------------------------------------------------
def _dense_inputs(k, hw=HW, seed=50, views=2, P=DENSE, **kw):
    sc = _with_culled(make_scene(P, views, *hw, seed=seed, **kw), k)
    cams, ins = _cams([sc])
    return cams, {n: ins[n] for n in ("means3D", "opacities", "shs", "cov3D_precomp")}


def test_interleaved_settings_on_one_shape():
    """Learned with anti-aliasing off and no depth; then on the same shape anti-aliasing, a depth mode, ALL_STRATA
    (which leaves the table to be reset), the warp-specialised compositor, and the default again."""
    hw = HW
    cams, ins = _dense_inputs(140)
    base = _plain_call(cams, hw)(ins)
    nf = _near_far(cams)
    calls = [base._replace(backward=False)] * 4 + [
        base._replace(bs=base.bs._replace(antialiasing=True), label="aa"),
        base._replace(bs=base.bs._replace(with_depth=True, depth_mode="log", depth_near_far=nf), label="log depth"),
        base._replace(ins=_faint(ins), bs=base.bs._replace(antialiasing=True), label="faint, aa"),
        base._replace(bs=base.bs._replace(tuning=ALL), label="all strata"),
        base._replace(ins=_faint(ins), bs=base.bs._replace(tuning=_capi.GS_TUNE_FWD_WS), label="fwd ws, faint"),
        base._replace(label="default"), base._replace(ins=_faint(ins), label="default, faint")]
    lazy = _identical("interleaved", _sequence(calls), atomic_calls=range(4, 11))
    assert all(r["stats"]["speculative"] == 2 for r in lazy[1:]), [r["stats"]["speculative"] for r in lazy]
    _oracle("interleaved, last call", calls[-1], lazy[-1], "plain")


def test_same_shape_key_different_frame():
    """64 x 80 and 80 x 64: the same V, P, S and 20 tiles, so one slot and one table, written by the other frame."""
    P = int(7.5 * 64 * 80)
    frames = []
    for hw in ((64, 80), (80, 64)):
        cams, ins = _dense_inputs(141, hw=hw, P=P, seed=51)
        frames.append(_plain_call(cams, hw)(ins))
    calls = []
    for i in range(10):
        c = frames[i % 2]
        calls.append(c._replace(ins=_faint(c.ins)) if i in (6, 7) else c)
    res = _sequence(calls, extras=(0, _capi.GS_TUNE_NO_SPECULATION))
    lazy = _identical("same key, two frames", res, atomic_calls=range(4, 10), ref_key=_capi.GS_TUNE_NO_SPECULATION)
    assert [r["stats"]["speculative"] for r in lazy][2:] == [2] * 8
    _oracle("same key, last call", calls[-1], lazy[-1], "plain")


def test_context_and_target_alternation():
    """One shape from two camera sets in turn: the table always comes from the other set."""
    hw = HW
    ca, ins = _dense_inputs(142, seed=52)
    cb, _ = _dense_inputs(142, seed=52, first_view=3, total_views=5)
    a, b = _plain_call(ca, hw)(ins), _plain_call(cb, hw)(ins)
    calls = [a, b] * 4 + [a._replace(ins=_faint(ins)), b._replace(ins=_faint(ins)), a]
    lazy = _identical("context / target", _sequence(calls), atomic_calls=range(4, 11))
    assert [r["stats"]["speculative"] for r in lazy][2:] == [2] * 9
    _oracle("context / target, faint", calls[-2], lazy[-2], "plain", faint=True)


def test_saved_state_across_a_lazy_re_sort():
    """Forward A (steady state, with grad); an identical forward A' and its backward; forward and backward B (same
    shape, faint: its compositor sorts strata); then A's backward.  A's gradients equal A''s, taken before B ran (bits
    for the deterministic backward), and those of the same sequence under ALL_STRATA -- the latter alone could not tell
    A reading B's fully sorted lists from A reading its own."""
    from pf3plat_b200.rasterizer import rasterize_batch
    hw = HW
    cams, ins = _dense_inputs(143, seed=53)
    c = _plain_call(cams, hw)(ins)
    inc = _incoming(c.bs)
    res = {}
    for extra in (0, ALL):
        s = torch.cuda.Stream(DEV)
        with torch.cuda.stream(s):
            for _ in range(4):
                _one(c._replace(backward=False), extra)
            bs = c.bs._replace(tuning=extra)
            la = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
            outa = rasterize_batch(bs, **la)
            ra2 = _one(c, extra)                                    # A', forward and backward before B
            rb = _one(c._replace(ins=_faint(ins)), extra)
            got = {}
            for det in (True, False):
                for t in la.values():
                    t.grad = None
                torch.use_deterministic_algorithms(det)
                try:
                    torch.autograd.backward([outa[0], outa[2]], [inc["color"], inc["alpha"]], retain_graph=det)
                finally:
                    torch.use_deterministic_algorithms(False)
                got[det] = {k: t.grad.clone() for k, t in la.items()}
            s.synchronize()
        res[extra] = (got, rb, ra2)
    for k in res[ALL][0][True]:
        assert torch.equal(res[0][0][True][k], res[0][2]["det"][k]), f"A's deterministic dL/d{k} differs from A''s"
        _close(f"A's atomic dL/d{k} vs A''s", res[0][0][False][k], res[0][2]["atomic"][k])
        assert torch.equal(res[0][0][True][k], res[ALL][0][True][k]), f"A's deterministic dL/d{k} differs"
        _close(f"A's atomic dL/d{k}", res[0][0][False][k], res[ALL][0][False][k])
        _close(f"A's atomic dL/d{k} vs deterministic", res[0][0][False][k], res[0][0][True][k])
        assert torch.equal(res[0][1]["det"][k], res[ALL][1]["det"][k]), f"B's deterministic dL/d{k} differs"
    print("[steady] saved state across a lazy re-sort: A's gradients bit-identical to A''s and to ALL_STRATA's")


def test_overflow_with_a_learned_table():
    """Call 5 moves 1.5x as many Gaussians again into the frame (the shape -- P -- is the same: they sat behind the
    camera): the speculative capacities overflow and the call is redone exactly.  The next two calls are correct and end
    back on strata.  (A cloud of 0.6 x the module's density, so that the redo's lists stay within the shared-memory sort
    and the call after it is the trial.)"""
    hw = HW
    n = int(0.6 * DENSE)
    sc = make_scene(int(2.5 * n), 2, *hw, seed=54)
    cams, ins = _cams([_with_culled(sc, 144)])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    behind = ins["means3D"].clone()
    behind[0, n:int(2.5 * n), 2] = -behind[0, n:int(2.5 * n), 2]
    c = _plain_call(cams, hw)
    small, big = c(dict(ins, means3D=behind)), c(ins)
    calls = [small._replace(backward=False)] * 4 + [big, small._replace(ins=_faint(small.ins)), small]
    res = _sequence(calls, extras=(0, ALL, _capi.GS_TUNE_NO_SPECULATION))
    lazy = _identical("overflow", res, atomic_calls=(4, 5, 6))
    _identical("overflow vs exact", {0: res[0], 1: res[_capi.GS_TUNE_NO_SPECULATION]}, atomic_calls=(), ref_key=1)
    spec = [r["stats"]["speculative"] for r in lazy]
    redos = [r["stats"]["overflow_redos"] for r in lazy]
    print(f"[steady] overflow: speculative {spec}, redos {redos}")
    assert spec == [0, 2, 2, 2, 0, 2, 2] and redos == [0, 0, 0, 0, 1, 1, 1], (spec, redos)
    _oracle("overflow, after the redo", calls[5], lazy[5], "plain", faint=True)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the training shape through decoder_forward
# ---------------------------------------------------------------------------------------------------------------------
def test_decoder_forward_at_the_training_shape(monkeypatch):
    """PF3plat's decoder call: b = 14 scenes x 3 views of 131 072 Gaussians at 256 x 256, extrinsics requiring grad, a
    colour and a depth loss; 6 steps, each moving the means by a small Adam-like step.  Each step's colour, depth and
    gradients equal the same steps under ALL_STRATA: bits for the deterministic backward, the atomic criterion for the
    default one."""
    from pf3plat_b200 import render
    from pf3plat_b200.rasterizer import last_stats
    b, v, G, hw = 14, 3, 131_072, (256, 256)
    scs = [make_scene(G, v, *hw, seed=900 + k) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs]).to(DEV)
    means0, cov, harm, opac = st("means"), st("covariances"), st("harmonics"), st("opacities")
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), 0.5, device=DEV), torch.full((b, v), 50.0, device=DEV)
    bg = torch.tensor([0.3, 0.2, 0.1], device=DEV)
    g = torch.Generator().manual_seed(901)
    # an Adam step moves every coordinate by about the learning rate: 1e-3 of a scene about 10 deep
    steps = [(torch.sign(torch.randn(means0.shape, generator=g)) * 1e-3).to(DEV) for _ in range(6)]
    dL = (torch.randn(b, v, 3, *hw, generator=g) / (b * v * hw[0] * hw[1])).to(DEV)
    wd = (torch.randn(b, v, *hw, generator=g) / (b * v * hw[0] * hw[1])).to(DEV)
    plain = render.rasterize_batch
    runs = {}
    for extra in (0, ALL):
        monkeypatch.setattr(render, "rasterize_batch", lambda bs, *a, **k: plain(bs._replace(tuning=bs.tuning | extra),
                                                                                  *a, **k))
        s = torch.cuda.Stream(DEV)
        out, stats = [], []
        with torch.cuda.stream(s):
            m = means0.clone()
            for k in range(6):
                m = m + steps[k]
                rec = {}
                for det in (True, False):
                    L = [t.clone().requires_grad_(True) for t in (m, cov, harm, opac)]
                    e = ext.clone().requires_grad_(True)
                    color, depth = render.decoder_forward(*L, e, intr, nr, fr, hw, bg, depth_mode="depth")
                    stats.append(last_stats(DEV))
                    torch.use_deterministic_algorithms(det)
                    try:
                        torch.autograd.backward([color, depth], [dL, wd])
                    finally:
                        torch.use_deterministic_algorithms(False)
                    rec[det] = ([color.detach(), depth.detach()], [t.grad.clone() for t in L] + [e.grad.clone()])
                out.append(rec)
            s.synchronize()
        runs[extra] = out
        spec, redos = [x["speculative"] for x in stats], [x["overflow_redos"] for x in stats]
        print(f"[steady] training shape (tuning {extra:#x}): speculative per forward {spec}, overflow redos {redos}")
        assert spec[1:] == [2] * 11 and redos == [0] * 12, (spec, redos)
    with torch.no_grad(), torch.cuda.stream(torch.cuda.Stream(DEV)):
        alpha = render.decoder_forward(means0, cov, harm, opac, ext, intr, nr, fr, hw, bg, return_alpha=True)[2]
        sat = float((alpha >= SAT).float().mean())
    print(f"[steady] training shape: saturated fraction {sat:.4f}")
    names = ("means", "covariances", "harmonics", "opacities", "extrinsics")
    for k in range(6):
        a, r = runs[0][k], runs[ALL][k]
        for det in (True, False):
            for x, y, n in zip(a[det][0], r[det][0], ("colour", "depth")):
                assert torch.equal(x, y), f"step {k + 1}: {n} differs"
        for x, y, n in zip(a[True][1], r[True][1], names):
            assert torch.equal(x, y), f"step {k + 1}: deterministic dL/d{n} differs"
        for x, y, n in zip(a[False][1], r[False][1], names):
            _close(f"step {k + 1}: atomic dL/d{n}", x, y)
            _close(f"step {k + 1}: atomic dL/d{n} vs deterministic", x, a[True][1][names.index(n)])
    print("[steady] training shape: 6 steps bit-identical to ALL_STRATA")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the production entries in the steady state: the host entry's feeds and the drop-in
# ---------------------------------------------------------------------------------------------------------------------
FEEDS = {"pageable upload": False, "pinned, zero-copy split colour pipeline": True}


@pytest.mark.parametrize("feed", list(FEEDS), ids=["pageable", "pinned-split"])
def test_host_entry_in_the_steady_state(feed):
    """gs_render_host_ex over five calls of one shape (dense x 3, moved, faint) on a context of its own: from the pinned
    buffers the default feed pulls the SH block zero-copy with k_sh_colour on a second stream, and the compositor --
    its lazy extension of the lists included -- waits for it on an event only.  Colour, radii and alpha are the bytes of
    the device entry on the same sequence, call by call, and both reach lazy strata from the second call on."""
    import ctypes
    from pf3plat_b200 import rasterizer
    from pf3plat_b200.rasterizer import _make_config, last_stats, rasterize_batch
    hw = HW
    pinned = FEEDS[feed]
    sc = _with_culled(make_scene(DENSE, 2, *hw, seed=62), 172 + pinned)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    moved = {k: v.cpu() for k, v in _moved(ins, hw, 63).items()}
    seq = [ins] * 3 + [moved, dict(ins, opacities=ins["opacities"] / 20)]
    V, P, M = 2, ins["means3D"].shape[1], ins["shs"].shape[2]
    bs_cpu = _settings(cams, hw, sh_degree=3)._replace(with_alpha=True, sh_eval_max_degree=3)
    bs_dev = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, sh_degree=3)._replace(with_alpha=True,
                                                                                          sh_eval_max_degree=3)
    ref, ref_spec = [], []
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s), torch.no_grad():
        for x in seq:
            out = rasterize_batch(bs_dev, **{k: v.to(DEV) for k, v in x.items()})
            ref.append([o.cpu() for o in out])
            ref_spec.append(last_stats(DEV)["speculative"])
        s.synchronize()
    keep: list = []
    cfg = _make_config(bs_cpu, 1, P, M, keep)
    color = torch.empty(V, 3, *hw).pin_memory()
    radii = torch.empty(V, P, dtype=torch.int32).pin_memory()
    alpha = torch.empty(V, *hw).pin_memory()
    gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr(), depth=None)
    req = _capi.GsAlpha(alpha.data_ptr(), None)
    spec = []
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        ctx = rasterizer.current_context(DEV)
        for i, x in enumerate(seq):
            host = {k: v[0].contiguous() for k, v in x.items()}
            if pinned:
                host = {k: v.pin_memory() for k, v in host.items()}
            gin = _capi.GsInputs(means3D=host["means3D"].data_ptr(), opacities=host["opacities"].data_ptr(),
                                 shs=host["shs"].data_ptr(), cov3D_precomp=host["cov3D_precomp"].data_ptr())
            color.zero_(); radii.zero_(); alpha.fill_(-1.0)
            _capi.check(_capi.lib().gs_render_host_ex(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                      ctypes.byref(req), s.cuda_stream))
            spec.append(last_stats(DEV)["speculative"])
            for name, got, want in (("colour", color, ref[i][0]), ("radii", radii, ref[i][1]), ("alpha", alpha, ref[i][2])):
                assert torch.equal(got, want), f"{feed} call {i + 1}: {name} differs from the device entry"
        s.synchronize()
    sat = [_saturation(bs_dev, {k: v.to(DEV) for k, v in x.items()}) for x in seq[2:]]
    print(f"[steady] host entry, {feed}: speculative per call {spec} (device entry {ref_spec}); saturated fraction "
          f"calls 3-4 {[round(x[0], 4) for x in sat[:2]]}, faint call 5 below alpha 0.999 {sat[2][1]:.4f}")
    assert spec == ref_spec == [0, 2, 2, 2, 2], (spec, ref_spec)
    assert min(x[0] for x in sat[:2]) >= 0.9 and sat[2][1] >= 0.9, sat


def test_dropin_in_the_steady_state(monkeypatch):
    """PF3plat's render_cuda call pattern (tests/ref_callsite.py: per-view GaussianRasterizer, S = V = 1, a zero means2D
    requiring grad) over five calls of one shape (dense x 3, moved, faint) with a colour loss: every image, radii and
    the deterministic backward's gradients (means2D included) equal the same calls under ALL_STRATA bit for bit, the
    atomic ones to the backward criterion, and the shape reaches lazy strata from the second call on."""
    from pf3plat_b200.rasterizer import GaussianRasterizer, last_stats
    from tests.ref_callsite import render_like_reference
    hw = HW
    sc = _with_culled(make_scene(DENSE, 1, *hw, seed=64), 174)
    g = torch.Generator().manual_seed(65)
    d = lambda t: t.to(DEV)
    cams = [d(sc.extrinsics), d(sc.intrinsics), d(sc.near), d(sc.far)]
    bgc = d(sc.background)
    px = sc.means[:, 2:3] * (2 * TANFOV / hw[1])
    moved = sc.means + torch.randn(sc.means.shape, generator=g) * px * torch.tensor([1.0, 1.0, 0.0])
    base = [d(sc.means[None]), d(sc.covariances[None]), d(sc.harmonics[None]), d(sc.opacities[None])]
    seq = [base] * 3 + [[d(moved[None])] + base[1:], base[:3] + [base[3] / 20]]
    dL = (torch.randn(1, 3, *hw, generator=g) / (hw[0] * hw[1])).to(DEV)
    plain = GaussianRasterizer._batch_settings
    runs = {}
    for extra in (0, ALL):
        monkeypatch.setattr(GaussianRasterizer, "_batch_settings",
                            lambda self, *a, **k: plain(self, *a, **k)._replace(tuning=extra))
        s = torch.cuda.Stream(DEV)
        rec, specs = [], []
        with torch.cuda.stream(s):
            for x in seq:
                got = {}
                for det in (True, False):
                    L = [t.clone().requires_grad_(True) for t in x]
                    img, radii, m2d = render_like_reference(*cams, hw, bgc, *L, return_radii=True, return_means2d=True)
                    specs.append(last_stats(DEV)["speculative"])
                    torch.use_deterministic_algorithms(det)
                    try:
                        img.backward(dL)
                    finally:
                        torch.use_deterministic_algorithms(False)
                    got[det] = [t.grad.clone() for t in L] + [m2d[0].grad.clone()]
                rec.append(([img.detach(), radii], got))
            s.synchronize()
        runs[extra] = rec
        print(f"[steady] drop-in (tuning {extra:#x}): speculative per forward {specs}")
        assert specs == [0] + [2] * 9, specs    # two forwards per call: one per backward
    names = ("means", "covariances", "harmonics", "opacities", "means2D")
    for i, ((out, got), (out0, got0)) in enumerate(zip(runs[0], runs[ALL])):
        for a, b, n in zip(out, out0, ("colour", "radii")):
            assert torch.equal(a, b), f"drop-in call {i + 1}: {n} differs"
        for a, b, n in zip(got[True], got0[True], names):
            assert torch.equal(a, b), f"drop-in call {i + 1}: deterministic dL/d{n} differs"
        for a, b, c, n in zip(got[False], got0[False], got[True], names):
            _close(f"drop-in call {i + 1}: atomic dL/d{n}", a, b)
            _close(f"drop-in call {i + 1}: atomic dL/d{n} vs deterministic", a, c)
    print("[steady] drop-in: 5 calls bit-identical to ALL_STRATA")
