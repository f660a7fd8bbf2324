"""GPU tests of anti-aliased rasterization (GS_FLAG_ANTIALIAS, BatchSettings.antialiasing, set_antialiasing): every splat
drawn at opacity o * rho, rho = sqrt(max(2.5e-5, det0 / det1)) of its projected covariance before / after the dilation,
with the gradient of rho carried into opacities, covariances or scales / rotations and means.

The oracle is tests/aa_oracle.py: per view, the fp64 oracle at opacities o * rho_v, rho_v from an fp64 autograd
restatement of the projection.  Images use the fragile-pixel rules of tests/util.py, gradients the element-wise rule
(check_grad).  Every test prints "[regime]" lines and asserts its regime was reached."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.aa_oracle import RATIO_MIN, AAOracle, _render_of
from tests.alpha_oracle import AlphaOracle
from tests.batch_oracle import scene_batch_args
from tests.depth_modes_oracle import DepthModeOracle
from tests.regimes import edge_straddle_scene, near_plane_scene, offscreen_scene, opaque_stack_scene
from tests.sh4_oracle import SH_BANDS4, ShOracleBatch, with_band4
from tests.test_antialias_cpu import _iso_settings, iso_centre
from tests.test_gpu_alpha import _Det, _f32
from tests.test_gpu_backward_paths import _stream_ctx
from tests.test_gpu_depth_chain import _depth_batch, _depth_field, _turned
from tests.test_gpu_regimes import _settings
from tests.util import FRAGILE_RGB_TOL, RGB_TOL, check_grad, check_image_strict

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEEP = ("means3D", "opacities", "shs", "cov3D_precomp")


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    """Contexts are cached per (device, stream) and torch reuses streams: start and end with none cached."""
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts, set_antialiasing
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    set_antialiasing(False)
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()


def _shrink(ins, every=3, factor=30.0):
    """Every `every`-th Gaussian `factor` times smaller (sub-pixel splats, rho << 1, next to large ones)."""
    out = dict(ins)
    P = ins["means3D"].shape[1]
    sel = torch.zeros(P, dtype=torch.bool)
    sel[::every] = True
    if "cov3D_precomp" in ins:
        c = ins["cov3D_precomp"].clone()
        c[:, sel] /= factor * factor
        out["cov3D_precomp"] = c
    if "scales" in ins:
        s = ins["scales"].clone()
        s[:, sel] /= factor
        out["scales"] = s
    return out


def _gpu(bs, ins, dL=None, w=None, dA=None, view_grad=False):
    """rasterize_batch with bs (device cameras) and a means2D sink; backward of <dL, colour> + <w, depth> + <dA, alpha>
    (None: left out of the loss).  Returns ({input: grad}, outputs, view-matrix grad)."""
    from pf3plat_b200.rasterizer import rasterize_batch
    vm = bs.viewmatrix.clone().requires_grad_(view_grad)
    V, P = bs.viewmatrix.shape[0], ins["means3D"].shape[1]
    leaves = {k: v.to(DEV).clone().requires_grad_(True) for k, v in ins.items()}
    leaves["means2D"] = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    out = rasterize_batch(bs._replace(viewmatrix=vm), **leaves)
    names = ["color", "radii"] + (["depth"] if bs.with_depth else []) + (["alpha"] if bs.with_alpha else [])
    o = dict(zip(names, out))
    ts, gs = [], []
    for key, g in (("color", dL), ("depth", w), ("alpha", dA)):
        if g is not None:
            ts.append(o[key])
            gs.append(_f32(g))
    if ts:
        torch.autograd.backward(ts, gs)
    return {k: t.grad for k, t in leaves.items()}, {k: v.detach() for k, v in o.items()}, vm.grad


def _check_images(label, color, orc, max_fragile=0.02):
    for v in range(orc.V):
        r = _render_of(orc.views[v])
        check_image_strict(color[v], r, max_fragile, f"{label} view {v}")


def _check_all_grads(label, grads, go, orc, bands=None):
    aff = orc.affected()
    VPS = orc.VPS
    for k, g in grads.items():
        if go.get(k) is None:
            assert g is None or float(g.abs().max()) == 0.0, k
            continue
        if k in ("colors_precomp", "means2D"):
            for v in range(g.shape[0]):
                check_grad(f"{label} dL/d{k} view {v}", g[v], go[k][v], aff[v // VPS])
        else:
            for s in range(g.shape[0]):
                check_grad(f"{label} dL/d{k} scene {s}", g[s].reshape(g.shape[1], -1) if k != "shs" else g[s],
                           go[k][s].reshape(g.shape[1], -1) if k != "shs" else go[k][s], aff[s],
                           bands if k == "shs" else None)


# ---------------------------------------------------------------------------------------------------------------------
# 1. against the oracle, under every compositor
# ---------------------------------------------------------------------------------------------------------------------
TUNINGS = ((0, "default"), (_capi.GS_TUNE_BWD_V1, "bwd v1"), (_capi.GS_TUNE_BWD_OCC4, "bwd occ4"),
           (_capi.GS_TUNE_FWD_WS, "warp-specialised fwd"))


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_aa_against_oracle_under_every_compositor(geometry):
    """S = 2 scenes x 9 views, view_scale 0.8 .. 1.25, turned cameras, every third Gaussian sub-pixel.  Colour + depth
    loss: images and every gradient against the oracle under both forward compositors and every backward compositor."""
    cams, ins, hw = _depth_batch(geometry)
    ins = _shrink(ins)
    V, S = cams["viewmatrix"].shape[0], 2
    bs_cpu = _settings(cams, hw, with_depth=True)._replace(antialiasing=True)
    orc = AAOracle(bs_cpu, ins)
    target = make_target(V, *hw, seed=3).numpy()
    dL = 2 * (orc.color - target) / target.size
    w = _depth_field(V, hw, 72)
    go = orc.backward(dL, w)
    vis = orc.radii > 0
    print(f"[regime] {geometry}: V={V}, rho of visible pairs {orc.rho[vis].min():.4f}..{orc.rho[vis].max():.4f} "
          f"({(orc.rho[vis] < 0.1).mean():.2f} below 0.1), affected {orc.affected().mean():.3f}")
    assert orc.rho[vis].min() < 0.05 and orc.rho[vis].max() > 0.9
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    for tuning, name in TUNINGS:
        bs = _settings(dcams, hw, with_depth=True, tuning=tuning)._replace(antialiasing=True)
        grads, out, _ = _gpu(bs, ins, dL=dL, w=w)
        _check_images(f"{geometry} {name}", out["color"], orc)
        derr = float(np.abs(out["depth"].cpu().double().numpy() - orc.depth).max())
        print(f"[parity] {geometry} {name}: depth max err {derr:.2e}")
        assert derr <= 1e-3 * float(np.abs(orc.depth).max())
        assert torch.equal(out["radii"].cpu(), torch.as_tensor(orc.radii))
        _check_all_grads(f"{geometry} {name}", grads, go, orc)


def test_aa_off_is_bit_identical_to_a_call_that_never_mentions_it():
    """antialiasing=False and the process-wide default give the bytes of a call without the field: colour, depth, alpha,
    radii and every gradient (deterministic mode); antialiasing=True changes colour and gradients but not radii."""
    from pf3plat_b200.rasterizer import BatchSettings
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    rng = np.random.default_rng(5)
    dL, w, dA = rng.standard_normal((V, 3, *hw)) / 1536, _depth_field(V, hw, 6), rng.standard_normal((V, *hw)) / 1536
    fields = {k: v for k, v in _settings(dcams, hw, with_depth=True)._asdict().items() if k != "antialiasing"}
    plain = BatchSettings(**fields)._replace(with_alpha=True)
    with _Det():
        ref = _gpu(plain, ins, dL=dL, w=w, dA=dA, view_grad=True)
        for label, bs in (("False", plain._replace(antialiasing=False)), ("None", plain._replace(antialiasing=None))):
            g, o, vg = _gpu(bs, ins, dL=dL, w=w, dA=dA, view_grad=True)
            for k in o:
                assert torch.equal(o[k], ref[1][k]), (label, k)
            for k in g:
                assert torch.equal(g[k], ref[0][k]), (label, k)
            assert torch.equal(vg, ref[2]), label
        g, o, _ = _gpu(plain._replace(antialiasing=True), ins, dL=dL, w=w, dA=dA, view_grad=True)
    assert torch.equal(o["radii"], ref[1]["radii"]) and not torch.equal(o["color"], ref[1]["color"])
    assert not torch.equal(g["opacities"], ref[0]["opacities"])
    print("[regime] anti-aliasing off: every output and gradient bit-identical to a call without the setting")


# ---------------------------------------------------------------------------------------------------------------------
# 2. binning paths: the same bits
# ---------------------------------------------------------------------------------------------------------------------
def test_aa_every_binning_path():
    """2 scenes x 3 views on a context of its own, walked through every binning state: images and the deterministic
    gradients are the exact path's bit for bit; the instance count falls against a call without anti-aliasing."""
    from pf3plat_b200.rasterizer import last_stats
    c = _capi
    hw = (32, 48)
    scenes = [make_scene(2500, 3, *hw, seed=80 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = _shrink({k: ins[k] for k in KEEP})
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    V = 6
    rng = np.random.default_rng(81)
    dL = rng.standard_normal((V, 3, *hw)) / 1536
    sequence = [("exact", c.GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("stratified, k_emit_buckets", c.GS_TUNE_SEPARATE_EMIT, 2),
                ("exact, re-learn unstratified", c.GS_TUNE_NO_STRATA | c.GS_TUNE_NO_SPECULATION, 0),
                ("whole-tile", c.GS_TUNE_NO_STRATA, 1), ("radix fallback", c.GS_TUNE_FORCE_RADIX_BINNING, 0)]
    stream = _stream_ctx(DEV)
    states, first, counts = [], None, []
    with torch.cuda.stream(stream), _Det():
        for label, tuning, want in sequence:
            bs = _settings(dcams, hw, tuning=tuning)._replace(antialiasing=True)
            grads, out, _ = _gpu(bs, ins, dL=dL)
            st = last_stats(DEV)
            states.append(st["speculative"])
            counts.append(st["num_rendered"])
            assert st["speculative"] == want and st["overflow_redos"] == 0, (label, st)
            if first is None:
                first = (grads, out)
            for k in out:
                assert torch.equal(out[k], first[1][k]), (label, k)
            for k in grads:
                assert torch.equal(grads[k], first[0][k]), (label, k)
        _gpu(_settings(dcams, hw, tuning=c.GS_TUNE_NO_SPECULATION), ins)
        plain = last_stats(DEV)["num_rendered"]
        stream.synchronize()
    print(f"[regime] AA binning paths: speculative per call {states}; instances {counts[0]} with AA, {plain} without")
    assert len(set(counts)) == 1 and counts[0] < plain


def test_aa_per_tile_strata_and_overflow_redo():
    """The pixel-aligned cloud (per-view strata trial overflows, then per-(view, tile) strata): images and deterministic
    gradients equal the exact path's."""
    from pf3plat_b200.rasterizer import last_stats
    sc = make_pixel_aligned_scene(128, 128, 3, seed=2)
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    dL = np.random.default_rng(82).standard_normal((3, 3, *hw)) / (hw[0] * hw[1])
    bs = lambda tuning=0: _settings(dcams, hw, tuning=tuning)._replace(antialiasing=True)
    with _Det():
        ref_g, ref, _ = _gpu(bs(_capi.GS_TUNE_NO_SPECULATION), ins, dL=dL)
        stream = _stream_ctx(DEV)
        states, redos = [], []
        with torch.cuda.stream(stream):
            for _ in range(5):
                grads, out, _ = _gpu(bs(), ins, dL=dL)
                st = last_stats(DEV)
                states.append(st["speculative"])
                redos.append(st["overflow_redos"])
                assert torch.equal(out["color"], ref["color"]), states
                for k in grads:
                    assert torch.equal(grads[k], ref_g[k]), (states, k)
            stream.synchronize()
    print(f"[regime] AA per-tile strata: speculative per call {states}, overflow redos {redos}")
    assert 2 in states and max(redos) >= 1


# ---------------------------------------------------------------------------------------------------------------------
# 3. option combinations: degree 4, every depth mode with the view-matrix gradient, alpha
# ---------------------------------------------------------------------------------------------------------------------
def _combo_batch(P=3000, hw=(40, 56), views=3, seed=13):
    sc = _turned(with_band4(make_scene(P, views, *hw, seed=seed)), seed=seed + 1)
    cams, ins = scene_batch_args([sc], near=1.0 / np.linspace(0.8, 1.25, views))
    return cams, _shrink({k: ins[k] for k in KEEP}), sc.image_shape


def test_aa_degree4():
    cams, ins, hw = _combo_batch()
    V = cams["viewmatrix"].shape[0]
    bs_cpu = _settings(cams, hw)._replace(antialiasing=True, sh_eval_max_degree=4)
    orc = AAOracle(bs_cpu, ins, view_oracle=lambda b, i: ShOracleBatch(b, i["means3D"], i["opacities"], i["shs"], deg=4,
                                                                       cov3D_precomp=i["cov3D_precomp"]))
    dL = np.random.default_rng(40).standard_normal((V, 3, *hw)) / (hw[0] * hw[1])
    go = orc.backward(dL)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    grads, out, _ = _gpu(_settings(dcams, hw)._replace(antialiasing=True, sh_eval_max_degree=4), ins, dL=dL)
    _check_images("degree 4", out["color"], orc)
    _check_all_grads("degree 4", grads, go, orc, bands=SH_BANDS4)
    print(f"[regime] AA degree 4: |dL/dsh band 4| max {np.abs(go['shs'][..., 16:25, :]).max():.2e}")
    assert np.abs(go["shs"][..., 16:25, :]).max() > 0


@pytest.mark.parametrize("mode", ["depth", "disparity", "relative_disparity", "log"])
def test_aa_every_depth_mode_with_the_view_matrix_gradient(mode):
    """Colour + depth loss in each depth mode: depth, the Gaussians' gradients and dL/dviewmatrix_z against the oracle of
    the reference's construction at the compensated opacities.  ("depth" composites the view-scaled z_s = s z: the oracle
    of z is scaled by s, and its incoming gradient with it.)"""
    cams, ins, hw = _combo_batch(seed=17)
    V = cams["viewmatrix"].shape[0]
    near = 1.0 / cams["view_scale"]
    nf = torch.stack([near, 100 * near], -1)
    s = cams["view_scale"].numpy().astype(np.float32).astype(np.float64)
    bs_cpu = _settings(cams, hw, with_depth=True)._replace(antialiasing=True, depth_mode=mode, depth_near_far=nf)
    orc = AAOracle(bs_cpu, ins, view_oracle=lambda b, i: DepthModeOracle(b, i, mode, b.depth_near_far))
    rng = np.random.default_rng(41)
    dL, w = rng.standard_normal((V, 3, *hw)) / 3072, _depth_field(V, hw, 42)
    f = s[:, None, None] if mode == "depth" else np.ones((V, 1, 1))
    go = orc.backward(dL, w * f)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)._replace(antialiasing=True, depth_mode=mode, depth_near_far=nf.to(DEV))
    grads, out, vg = _gpu(bs, ins, dL=dL, w=w, view_grad=True)
    _check_images(f"depth mode {mode}", out["color"], orc)
    want_depth = orc.depth * f
    derr = float(np.abs(out["depth"].cpu().double().numpy() - want_depth).max())
    print(f"[parity] AA depth mode {mode}: depth max err {derr:.2e} of {np.abs(want_depth).max():.2e}")
    assert derr <= 1e-3 * max(float(np.abs(want_depth).max()), 1e-6)
    grads.pop("means2D")
    _check_all_grads(f"depth mode {mode}", {k: g for k, g in grads.items() if k != "shs"}, go, orc)
    got_vz = vg.reshape(V, 16)[:, [2, 6, 10, 14]].cpu().double().numpy()
    scale = np.abs(go["view_z"]).max()
    err = np.abs(got_vz - go["view_z"]).max()
    print(f"[parity] AA depth mode {mode}: dL/dviewmatrix_z max err {err:.2e} of {scale:.2e}")
    assert err <= 1e-3 * scale + 1e-9
    if mode != "log":
        assert scale > 0


def test_aa_with_alpha():
    cams, ins, hw = _combo_batch(seed=19)
    V = cams["viewmatrix"].shape[0]
    bs_cpu = _settings(cams, hw)._replace(antialiasing=True, with_alpha=True)
    orc = AAOracle(bs_cpu, ins, view_oracle=lambda b, i: AlphaOracle(b, i))
    rng = np.random.default_rng(43)
    dA, dL = rng.standard_normal((V, *hw)) / 3072, rng.standard_normal((V, 3, *hw)) / 3072
    go = orc.backward(dA, dL)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    grads, out, _ = _gpu(_settings(dcams, hw)._replace(antialiasing=True, with_alpha=True), ins, dL=dL, dA=dA)
    _check_images("alpha", out["color"], orc)
    err = np.abs(out["alpha"].cpu().double().numpy() - orc.stack("alpha"))
    frag = orc.stack("frag")
    print(f"[parity] AA alpha: max err non-fragile {err[~frag].max():.2e}")
    assert err[~frag].max() <= RGB_TOL and (not frag.any() or err[frag].max() <= FRAGILE_RGB_TOL)
    _check_all_grads("alpha", grads, go, orc)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the host entry
# ---------------------------------------------------------------------------------------------------------------------
def test_host_entry_returns_the_device_entry_bytes():
    """Every feed of gs_render_host / gs_render_host_ex with GS_FLAG_ANTIALIAS returns the device entry's bytes."""
    from pf3plat_b200 import rasterizer
    P, V, hw = 20000, 3, (64, 80)
    sc = make_scene(P, V, *hw, seed=14)
    cams, ins = scene_batch_args([sc])
    ins = _shrink({k: ins[k] for k in KEEP})
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    ref = _gpu(_settings(dcams, hw, with_depth=True)._replace(with_alpha=True, antialiasing=True), ins)[1]
    host = {k: v[0].contiguous() for k, v in ins.items()}
    M = host["shs"].shape[1]
    cfg = _capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = P, 1, V, M, 4
    cfg.image_height, cfg.image_width, cfg.scale_modifier = hw[0], hw[1], 1.0
    cfg.flags = _capi.GS_FLAG_DEPTH | _capi.GS_FLAG_ANTIALIAS
    hc = {k: v.contiguous() for k, v in cams.items()}
    for k, t in hc.items():
        setattr(cfg, k, t.data_ptr())
    ctx = rasterizer.current_context(DEV)
    color = torch.empty(V, 3, *hw).pin_memory()
    radii = torch.empty(V, P, dtype=torch.int32).pin_memory()
    depth = torch.empty(V, *hw).pin_memory()
    alpha = torch.empty(V, *hw).pin_memory()
    gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr(), depth=depth.data_ptr())
    pin = {k: v.pin_memory() for k, v in host.items()}
    runs = 0
    for src in (host, pin):
        gin = _capi.GsInputs(means3D=src["means3D"].data_ptr(), opacities=src["opacities"].data_ptr(),
                             shs=src["shs"].data_ptr(), cov3D_precomp=src["cov3D_precomp"].data_ptr())
        feeds = (0, _capi.GS_TUNE_DIRECT_OUTPUT) if src is host else \
            (0, _capi.GS_TUNE_NO_SPLIT_COLOUR, _capi.GS_TUNE_NO_ZERO_COPY, _capi.GS_TUNE_DIRECT_OUTPUT)
        for tuning in feeds:
            for with_alpha in (False, True):
                cfg.tuning = tuning
                color.zero_(); radii.zero_(); depth.zero_(); alpha.fill_(-1.0)
                stream = torch.cuda.current_stream(DEV).cuda_stream
                if with_alpha:
                    rc = _capi.lib().gs_render_host_ex(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                       ctypes.byref(_capi.GsAlpha(alpha.data_ptr(), None)), stream)
                else:
                    rc = _capi.lib().gs_render_host(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), stream)
                _capi.check(rc)
                assert torch.equal(color, ref["color"].cpu()) and torch.equal(radii, ref["radii"].cpu()), tuning
                assert torch.equal(depth, ref["depth"].cpu()), tuning
                if with_alpha:
                    assert torch.equal(alpha, ref["alpha"].cpu()), tuning
                runs += 1
    print(f"[regime] AA host entry: M = {M}, {runs} runs bit-identical to the device entry")
    assert M > 16 and runs == 12


# ---------------------------------------------------------------------------------------------------------------------
# 5. regimes: closed form, sub-pixel clouds, large footprints, faint splats, edge cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sigma", [0.01, 0.05, 0.1, 0.5, 1.0, 3.0])
def test_closed_form_centre_pixel(sigma):
    from pf3plat_b200.rasterizer import rasterize_batch
    for opacity in (0.6, 1.0):
        bs, ins = _iso_settings(sigma, opacity)
        bs = bs._replace(**{k: getattr(bs, k).float().to(DEV) for k in ("viewmatrix", "projmatrix", "campos", "bg")})
        with torch.no_grad():
            out = rasterize_batch(bs, **{k: v.float().to(DEV) for k, v in ins.items()})
        got = out[0][0, :, 16, 16].cpu().double().numpy()
        want = iso_centre(sigma, opacity)
        print(f"[parity] sigma {sigma} px, o {opacity}: centre {got}, closed form {want}")
        assert np.abs(got - want).max() <= 1e-5


def _regime(label, sc, tuning=0, max_fragile=0.02, transform=None):
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    if transform is not None:
        ins = transform(ins)
    V = cams["viewmatrix"].shape[0]
    orc = AAOracle(_settings(cams, hw)._replace(antialiasing=True), ins)
    dL = np.random.default_rng(79).standard_normal((V, 3, *hw)) / (hw[0] * hw[1])
    go = orc.backward(dL)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    grads, out, _ = _gpu(_settings(dcams, hw, tuning=tuning)._replace(antialiasing=True), ins, dL=dL)
    _check_images(label, out["color"], orc, max_fragile)
    _check_all_grads(label, grads, go, orc)
    return orc, out


def _scaled_cov(f):
    def t(ins):
        out = dict(ins)
        out["cov3D_precomp"] = ins["cov3D_precomp"] * f
        return out
    return t


def test_sub_pixel_cloud_at_the_clamp():
    """sigma ~ 0.05 px: rho on both sides of its clamp."""
    sc = make_scene(1500, 2, 40, 56, seed=50)
    orc, _ = _regime("sub-pixel cloud", sc, transform=_scaled_cov(3e-3))
    vis = orc.radii > 0
    at = float((orc.ratio[vis] <= RATIO_MIN).mean())
    print(f"[regime] sub-pixel: rho {orc.rho[vis].min():.4f}..{orc.rho[vis].max():.4f}, at the clamp {at:.2f}, "
          f"within 0.1 % of it {orc.near_clamp[vis].sum()} pairs")
    assert 0.2 < at < 0.8 and np.median(orc.rho[vis]) < 0.05


def test_large_footprints():
    sc = make_scene(800, 2, 40, 56, seed=51)
    # (footprints this large overlap heavily: more pixels sit at an undecided 1/255 or T < 1e-4 threshold)
    orc, _ = _regime("large footprints", sc, transform=_scaled_cov(25.0), max_fragile=0.05)
    vis = orc.radii > 0
    print(f"[regime] large footprints: median rho {np.median(orc.rho[vis]):.4f}")
    assert np.median(orc.rho[vis]) > 0.95


def test_splats_whose_compensated_opacity_falls_below_the_threshold():
    """o * rho < 1/255: the radius is reported but the splat joins no tile and changes no pixel."""
    from pf3plat_b200.rasterizer import last_stats
    sc = make_scene(1200, 2, 40, 56, seed=52)

    def faint(ins):
        out = _scaled_cov(1e-3)(ins)
        out["opacities"] = ins["opacities"] * 0.5
        return out
    orc, out = _regime("faint splats", sc, transform=faint)
    vis = orc.radii > 0
    o = orc.opac[0][None] * orc.rho
    below = vis & (o < 1 / 255)
    print(f"[regime] faint splats: {below.sum()} visible pairs with o * rho < 1/255 of {vis.sum()}")
    assert below.sum() > 50
    assert torch.equal(out["radii"].cpu(), torch.as_tensor(orc.radii))
    # the tile instances are those of the splats above the threshold: never more than the oracle's 3-sigma squares hold
    assert last_stats(DEV)["num_rendered"] <= sum(_render_of(v).num_rendered for v in orc.views)


@pytest.mark.parametrize("hw", [(1, 40), (33, 250)])
def test_thin_and_ragged_frames(hw):
    sc = _turned(edge_straddle_scene(600, 120, 2, *hw, seed=90), seed=91)
    _regime(f"{hw[0]} x {hw[1]} frame", sc, transform=lambda i: _shrink(i))


@pytest.mark.parametrize("tuning", [0, _capi.GS_TUNE_FWD_WS | _capi.GS_TUNE_BWD_V1])
def test_opaque_stacks(tuning):
    sc = opaque_stack_scene(6, 12, 2, 48, 64, seed=93)
    orc, _ = _regime("opaque stack", sc, tuning=tuning, max_fragile=0.2)
    assert float((np.stack([_render_of(v).final_T for v in orc.views]) < 1e-3).mean()) > 0.1


def test_offscreen_and_near_plane():
    _regime("off-screen", offscreen_scene(1500, 200, 2, 48, 64, seed=94), transform=lambda i: _shrink(i))
    _regime("near plane", near_plane_scene(1500, 40, 40, 40, 2, 48, 64, seed=95), max_fragile=0.05)


def test_several_scenes_and_19_views_per_scene():
    hw = (24, 32)
    scenes = [make_scene(700, 19, *hw, seed=60 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 19), 2))
    ins = _shrink({k: ins[k] for k in KEEP})
    V = cams["viewmatrix"].shape[0]
    orc = AAOracle(_settings(cams, hw)._replace(antialiasing=True), ins)
    dL = np.random.default_rng(61).standard_normal((V, 3, *hw)) / (hw[0] * hw[1])
    go = orc.backward(dL)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    grads, out, _ = _gpu(_settings(dcams, hw)._replace(antialiasing=True), ins, dL=dL)
    _check_images("2 scenes x 19 views", out["color"], orc)
    _check_all_grads("2 scenes x 19 views", grads, go, orc)
    print(f"[regime] S = 2, {V // 2} views per scene")


# ---------------------------------------------------------------------------------------------------------------------
# 6. the drop-in and the decoder
# ---------------------------------------------------------------------------------------------------------------------
def test_dropin_through_the_reference_call_site():
    """tests/ref_callsite.py (render_cuda line by line) with set_antialiasing(True) equals the batched entry with
    antialiasing=True; a backward run after the setting was switched off still differentiates the anti-aliased forward."""
    from pf3plat_b200.rasterizer import set_antialiasing
    from pf3plat_b200.render import render_views
    from tests.ref_callsite import render_like_reference
    hw = (48, 64)
    sc = make_scene(3000, 2, *hw, seed=96).to(DEV)
    args = lambda: (sc.extrinsics, sc.intrinsics, sc.near, sc.far, hw, sc.background)
    target = make_target(2, *hw, seed=4).to(DEV)

    def run(fn, aa_forward, aa_backward, **kw):
        m = sc.means[None].repeat(2, 1, 1).clone().requires_grad_(True)
        o = sc.opacities[None].repeat(2, 1).clone().requires_grad_(True)
        cov = sc.covariances[None].repeat(2, 1, 1, 1)
        set_antialiasing(aa_forward)
        img = fn(*args(), m, cov, sc.harmonics[None].repeat(2, 1, 1, 1), o, **kw)
        set_antialiasing(aa_backward)
        ((img - target) ** 2).mean().backward()
        set_antialiasing(False)
        return img.detach(), m.grad, o.grad

    with _Det():
        on = run(render_like_reference, True, True)
        switched = run(render_like_reference, True, False)
        off = run(render_like_reference, False, False)
        batched = run(render_views, False, False, antialiasing=True)
    for a, b in zip(on, switched):
        assert torch.equal(a, b)
    assert not torch.equal(on[0], off[0]) and not torch.equal(on[2], off[2])
    err = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30) for a, b in zip(on[1:], batched[1:]))
    print(f"[regime] drop-in with set_antialiasing(True): image max |ref call site - batched| "
          f"{float((on[0] - batched[0]).abs().max()):.2e}, gradients rel {err:.2e}")
    assert float((on[0] - batched[0]).abs().max()) <= 1e-5 and err <= 1e-3


def test_decoder_forward_at_pf3plat_shape():
    """b = 14, v = 3, 131072 Gaussians per scene, 256^2, depth_mode "depth" on poses that require grad: anti-aliasing
    changes the images and lowers the instance count; antialiasing=False is the default call's bytes."""
    from pf3plat_b200 import render
    from pf3plat_b200.rasterizer import last_stats
    b, v, P, hw = 14, 3, 131072, (256, 256)
    g = torch.Generator(device="cpu").manual_seed(7)
    means = torch.randn(b, P, 3, generator=g) * torch.tensor([1.5, 1.5, 0.8]) + torch.tensor([0.0, 0.0, 5.0])
    A = torch.randn(b, P, 3, 3, generator=g) * 0.01
    cov = (A @ A.transpose(-1, -2) + 1e-5 * torch.eye(3)).to(DEV)
    harm = (torch.randn(b, P, 3, 25, generator=g) * 0.2).to(DEV)
    opac = torch.rand(b, P, generator=g).to(DEV)
    means = means.to(DEV)
    ext = torch.eye(4).repeat(b, v, 1, 1)
    ext[..., 0, 3] = torch.linspace(-0.2, 0.2, v)
    ext = ext.to(DEV)
    intr = torch.tensor([[1.0, 0, 0.5], [0, 1.0, 0.5], [0, 0, 1]]).repeat(b, v, 1, 1).to(DEV)
    nr, fr = torch.full((b, v), 0.5, device=DEV), torch.full((b, v), 100.0, device=DEV)
    bg = torch.zeros(3, device=DEV)
    res = {}
    for aa in (None, False, True):
        e = ext.clone().requires_grad_(True)
        m = means.clone().requires_grad_(True)
        color, depth = render.decoder_forward(m, cov, harm, opac, e, intr, nr, fr, hw, bg, depth_mode="depth",
                                              antialiasing=aa)
        n = last_stats(DEV)["num_rendered"]
        (color.square().mean() + depth.mean()).backward()
        res[aa] = (color.detach(), depth.detach(), e.grad, m.grad, n)
    assert torch.equal(res[None][0], res[False][0]) and torch.equal(res[None][1], res[False][1])
    assert res[None][4] == res[False][4]
    c, d, eg, mg, n = res[True]
    assert not torch.equal(c, res[None][0]) and torch.isfinite(eg).all() and float(eg.abs().max()) > 0
    assert torch.isfinite(mg).all() and n < res[None][4]
    print(f"[regime] decoder at PF3plat's shape: instances {res[None][4]} -> {n} with anti-aliasing")
