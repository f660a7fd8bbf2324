"""CPU checks of anti-aliased rasterization (GS_FLAG_ANTIALIAS): the fp64 composition oracle of tests/aa_oracle.py against
an independent autograd restatement (oracle/torch_oracle.py drawing each splat at o * rho, rho built by autograd) and
against finite differences; a closed-form centre pixel; rho at and on both sides of its clamp; rho against the dilated
covariance the C oracle's conic implies; and the C-ABI and Python pieces -- the flag, gs_supported_flags(), the knobs the
library refuses with the flag, the unchanged ABI, the BatchSettings field placement."""
import ctypes
import inspect
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import torch_oracle
from pf3plat_b200.synthetic import make_scene
from tests.aa_oracle import RATIO_MIN, AAOracle, aa_ratio, aa_rho, cov2d, sigma3
from tests.batch_oracle import batch_view_settings, oracle_batch, scene_batch_args
from tests.util import simple_settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _batch(geometry, views=2, seed=5, P=300, hw=(32, 48), use_sh=True):
    """One scene seen by `views` cameras with view_scale 0.8 .. 1.25; every third Gaussian shrunk 30x so that sub-pixel
    splats (rho << 1) are present next to large ones (rho -> 1)."""
    from pf3plat_b200.rasterizer import BatchSettings
    sc = make_scene(P, views, *hw, seed=seed)
    cams, ins = scene_batch_args([sc], near=1.0 / np.linspace(0.8, 1.25, views), use_sh=use_sh)
    small = torch.zeros(P, dtype=torch.bool)
    small[::3] = True
    ins["cov3D_precomp"][:, small] /= 900.0
    ins["scales"][:, small] /= 30.0
    keep = ("means3D", "opacities") + (("shs",) if use_sh else ()) + \
        (("cov3D_precomp",) if geometry == "cov3D" else ("scales", "rotations"))
    ins = {k: ins[k].double() for k in keep}
    if not use_sh:
        ins["colors_precomp"] = torch.rand(views, P, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=cams["viewmatrix"], projmatrix=cams["projmatrix"],
                       campos=cams["campos"], bg=cams["bg"], sh_degree=3, tanfov=cams["tanfov"],
                       view_scale=cams["view_scale"], antialiasing=True)
    return bs, ins


def _torch_aa(bs, ins, w):
    """<w, colour> of the anti-aliased render by autograd alone: per view, torch_oracle.render at opacities o * rho_v with
    rho_v built from the same leaves.  Returns (images [V,3,H,W], {input: grad})."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
    V, S = int(bs.viewmatrix.shape[0]), leaves["means3D"].shape[0]
    vps = V // S
    s_all = bs.view_scale.numpy().astype(np.float32).astype(np.float64)
    M = leaves["shs"].shape[2] if "shs" in leaves else 0
    loss, imgs = 0.0, []
    for v in range(V):
        k, s = v // vps, float(s_all[v])
        st = batch_view_settings(bs, v, M)
        m = leaves["means3D"][k] * s
        a0, b, c0 = cov2d(st, m, sigma3(leaves, k) * (s * s))
        kw = {"means3D": m, "opacities": leaves["opacities"][k] * aa_rho(aa_ratio(a0, b, c0, st.dilation))}
        if "shs" in leaves:
            kw["shs"] = leaves["shs"][k]
        else:
            kw["colors_precomp"] = leaves["colors_precomp"][v]
        if "cov3D_precomp" in leaves:
            kw["cov3D_precomp"] = leaves["cov3D_precomp"][k] * (s * s)
        else:
            kw["scales"], kw["rotations"] = leaves["scales"][k] * s, leaves["rotations"][k]
        color, _ = torch_oracle.render(st, **kw)
        imgs.append(color.detach().numpy())
        loss = loss + (color * torch.as_tensor(w[v])).sum()
    loss.backward()
    return np.stack(imgs), {k: t.grad.numpy() for k, t in leaves.items()}


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_composition_matches_the_autograd_restatement(geometry):
    bs, ins = _batch(geometry)
    orc = AAOracle(bs, ins)
    V = orc.V
    w = np.random.default_rng(1).standard_normal(orc.color.shape)
    imgs, want = _torch_aa(bs, ins, w)
    vis = orc.radii > 0
    print(f"[regime] {geometry}: rho of visible pairs {orc.rho[vis].min():.4f}..{orc.rho[vis].max():.4f}, "
          f"{(orc.rho[vis] < 0.1).mean():.2f} below 0.1, max |composition - autograd| image "
          f"{np.abs(imgs - orc.color).max():.2e}")
    assert orc.rho[vis].min() < 0.05 and orc.rho[vis].max() > 0.9
    np.testing.assert_allclose(orc.color, imgs, rtol=0, atol=1e-12)
    g = orc.backward(w)
    for k, t in want.items():
        got = g[k].reshape(t.shape) if k != "colors_precomp" else g[k]
        scale, err = np.abs(t).max(), np.abs(got - t).max()
        print(f"[parity] {geometry} dL/d{k}: max |composition - autograd| {err:.2e} of {scale:.2e}")
        assert scale > 0 and err <= 1e-6 * scale, k
    # without the compensation the opacity gradient would be dL/do', not rho dL/do'
    plain = oracle_batch(bs, dtype=np.float64, **ins).backward(w)
    assert np.abs(plain["opacities"] - g["opacities"]).max() > 1e-3 * np.abs(g["opacities"]).max()


def test_composition_matches_finite_differences():
    """Directional derivatives of <w, colour> in fp64 along random directions of the opacities, means and covariances of
    the Gaussians at no fragile decision and away from the clamp."""
    bs, ins = _batch("cov3D", views=2, seed=9, P=240, use_sh=False)
    orc = AAOracle(bs, ins)
    w = np.random.default_rng(2).standard_normal(orc.color.shape)
    g = orc.backward(w)
    safe = ~orc.affected()[0]
    rng = np.random.default_rng(3)
    P = ins["means3D"].shape[1]

    def loss(inputs):
        return float((AAOracle(bs, inputs).color * w).sum())

    for k, h in (("opacities", 1e-7), ("means3D", 1e-7), ("cov3D_precomp", 1e-9)):
        d = rng.standard_normal(ins[k].shape) * safe.reshape((1, P) + (1,) * (ins[k].dim() - 2))
        fd = (loss({**ins, k: ins[k] + h * torch.as_tensor(d)}) - loss({**ins, k: ins[k] - h * torch.as_tensor(d)})) / (2 * h)
        an = float((g[k].reshape(d.shape) * d).sum())
        print(f"[parity] finite differences dL/d{k}: analytic {an:.6e}, central difference {fd:.6e}")
        assert abs(an) > 0 and abs(fd - an) <= 1e-5 * abs(an), k


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_rho_matches_the_dilated_covariance_of_the_c_oracle(geometry):
    bs, ins = _batch(geometry, views=3, seed=11)
    orc = AAOracle(bs, ins)
    worst = orc.check_conic()
    print(f"[parity] {geometry}: restated (a0 + h, b, c0 + h) against the C oracle's conic, max rel {worst:.2e}")
    assert worst < 1e-9


def _iso_settings(sigma_px, opacity, colour=(0.8, 0.3, 0.1), bg=(0.2, 0.4, 0.6)):
    """An isotropic Gaussian on the optical axis of a 33 x 33 camera (centre pixel 16, 16) whose projected sigma is
    sigma_px pixels."""
    from pf3plat_b200.rasterizer import BatchSettings
    st = simple_settings(h=33, w=33, tanfov=0.5, bg=bg)
    z, f = 5.0, 33.0
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)[None]
    bs = BatchSettings(image_height=33, image_width=33, viewmatrix=t(st.viewmatrix), projmatrix=t(st.projmatrix),
                       campos=t(st.campos), bg=t(st.bg), sh_degree=0, tanfovx=0.5, tanfovy=0.5, antialiasing=True)
    sw = sigma_px * z / f
    ins = {"means3D": torch.tensor([[[0.0, 0.0, z]]], dtype=torch.float64),
           "opacities": torch.tensor([[opacity]], dtype=torch.float64),
           "colors_precomp": torch.tensor([[colour]], dtype=torch.float64),
           "cov3D_precomp": torch.tensor([[[sw * sw, 0, 0, sw * sw, 0, sw * sw]]], dtype=torch.float64)}
    return bs, ins


def iso_centre(sigma_px, opacity, colour=(0.8, 0.3, 0.1), bg=(0.2, 0.4, 0.6)):
    """min(0.99, o sigma^2 / (sigma^2 + 0.3)) c + (1 - alpha) bg, with rho's clamp (the closed form the tests expect)."""
    s2 = sigma_px ** 2
    a = min(0.99, opacity * max(s2 / (s2 + 0.3), np.sqrt(RATIO_MIN)))
    a = a if a >= 1 / 255 else 0.0
    return a * np.asarray(colour) + (1 - a) * np.asarray(bg)


@pytest.mark.parametrize("sigma", [0.05, 0.1, 0.5, 1.0, 3.0])
@pytest.mark.parametrize("opacity", [0.6, 1.0])
def test_closed_form_centre_pixel(sigma, opacity):
    bs, ins = _iso_settings(sigma, opacity)
    orc = AAOracle(bs, ins)
    got = orc.color[0, :, 16, 16]
    want = iso_centre(sigma, opacity)
    print(f"[parity] sigma {sigma} px, o {opacity}: rho {orc.rho[0, 0]:.5f}, centre {got}, closed form {want}")
    np.testing.assert_allclose(orc.rho[0, 0], sigma ** 2 / (sigma ** 2 + 0.3), rtol=1e-9)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def test_rho_at_and_around_its_clamp():
    # the isotropic sigma whose ratio sits exactly at the clamp: (s2 / (s2 + h))^2 = 2.5e-5
    r = np.sqrt(RATIO_MIN)
    s2 = 0.3 * r / (1 - r)
    for f, above in ((1 - 1e-6, False), (1.0, False), (1 + 1e-6, True)):
        a0 = torch.tensor(s2 * f, dtype=torch.float64, requires_grad=True)
        ratio = aa_ratio(a0, torch.tensor(0.0, dtype=torch.float64), a0, 0.3)
        rho = aa_rho(ratio)
        rho.backward()
        print(f"[regime] ratio / clamp = {float(ratio) / RATIO_MIN:.8f}: rho {float(rho):.8f}, drho/da0 {float(a0.grad):.4e}")
        assert abs(float(rho) - np.sqrt(max(float(ratio), RATIO_MIN))) < 1e-15
        assert (float(a0.grad) > 0) == above   # a constant below and at the clamp, growing above it
    assert float(aa_rho(torch.tensor(0.0, dtype=torch.float64))) == np.sqrt(RATIO_MIN)
    assert float(aa_rho(torch.tensor(-1.0, dtype=torch.float64))) == np.sqrt(RATIO_MIN)   # degenerate covariance
    # a splat far below the clamp: drawn at o * 0.005, and its gradient carries no rho term
    bs, ins = _iso_settings(0.01, 1.0)
    orc = AAOracle(bs, ins)
    assert orc.ratio[0, 0] < RATIO_MIN and orc.rho[0, 0] == np.sqrt(RATIO_MIN)
    g = orc.backward(np.ones((1, 3, 33, 33)))
    base = oracle_batch(bs, dtype=np.float64, **{**ins, "opacities": ins["opacities"] * np.sqrt(RATIO_MIN)}).backward(
        np.ones((1, 3, 33, 33)))
    np.testing.assert_allclose(g["cov3D_precomp"], base["cov3D_precomp"], rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------------------------------
# the C ABI and the Python surface
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_flag_and_supported_flags_match_the_header(capi, tmp_path):
    prog = tmp_path / "aa.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\n'
                    '_Static_assert(__builtin_types_compatible_p(__typeof__(&gs_supported_flags), uint32_t (*)(void)), '
                    '"gs_supported_flags prototype");\n'
                    'int main(void){printf("%u %u %u %u %d %zu %zu %zu\\n", (unsigned)GS_FLAG_ANTIALIAS, (unsigned)GS_FLAG_DEPTH,'
                    '(unsigned)GS_FLAG_PREFILTERED, (unsigned)GS_FLAG_DETERMINISTIC, GS_ABI_VERSION, sizeof(GsConfig),'
                    'sizeof(GsOutputs), sizeof(GsOutGrads));return 0;}')
    exe = tmp_path / "aa"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert out[0] == capi.GS_FLAG_ANTIALIAS == 8
    assert out[1:4] == [capi.GS_FLAG_DEPTH, capi.GS_FLAG_PREFILTERED, capi.GS_FLAG_DETERMINISTIC]
    assert out[4] == capi.ABI_VERSION == 5
    assert out[5:] == [ctypes.sizeof(capi.GsConfig), ctypes.sizeof(capi.GsOutputs), ctypes.sizeof(capi.GsOutGrads)]
    L = capi.lib()
    assert capi.SYMBOLS["gs_supported_flags"] == (ctypes.c_uint32, [])
    assert L.gs_supported_flags.restype is ctypes.c_uint32
    assert L.gs_supported_flags() == out[0] | out[1] | out[2] | out[3]


def _request(capi, tuning, flags):
    """A request that is valid in every respect but the anti-aliasing one (device pointers are never dereferenced)."""
    fake = 256
    cfg = capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = 16, 1, 1, 0, 0
    cfg.image_height, cfg.image_width, cfg.scale_modifier = 16, 16, 1.0
    cfg.viewmatrix = cfg.projmatrix = cfg.campos = cfg.bg = fake
    cfg.flags, cfg.tuning = flags, tuning
    gin = capi.GsInputs(means3D=fake, opacities=fake, colors_precomp=fake, cov3D_precomp=fake)
    gout = capi.GsOutputs(color=fake, radii=fake)
    return cfg, gin, gout


@pytest.mark.parametrize("knob", ["GS_TUNE_PRE_OCC6", "GS_TUNE_PBWD_2PHASE"])
def test_knobs_without_an_anti_aliased_kernel_are_refused(capi, knob):
    L = capi.lib()
    cfg, gin, gout = _request(capi, getattr(capi, knob), capi.GS_FLAG_ANTIALIAS)
    fake = ctypes.c_void_p(256)
    saved = ctypes.c_void_p(1234)
    assert L.gs_forward(fake, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), ctypes.byref(saved), None) == -1
    assert knob.encode() in L.gs_last_error() and b"GS_FLAG_ANTIALIAS" in L.gs_last_error()
    assert L.gs_render_host(fake, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), None) == -1
    assert knob.encode() in L.gs_last_error()
    if knob == "GS_TUNE_PBWD_2PHASE":   # (the other knob is the forward's: a backward goes on with it, so it is not called)
        og, ig = capi.GsOutGrads(256, None), capi.GsInGrads()
        rc = L.gs_backward(fake, ctypes.byref(cfg), ctypes.byref(gin), fake, ctypes.byref(og), ctypes.byref(ig), None)
        assert rc == -1 and knob.encode() in L.gs_last_error()


def test_batch_settings_and_entry_points():
    from pf3plat_b200 import rasterizer
    from pf3plat_b200.render import decoder_forward, render_views
    from pf3plat_b200.rasterizer import BatchSettings, GaussianRasterizationSettings, GaussianRasterizer
    f = BatchSettings._fields
    assert f[-1] == "with_alpha" and f[-2] == "antialiasing" and BatchSettings._field_defaults["antialiasing"] is None
    assert f.index("depth_near_far") == f.index("antialiasing") - 1
    assert len(GaussianRasterizationSettings._fields) == 12
    for fn in (GaussianRasterizer.forward, render_views, decoder_forward):
        assert inspect.signature(fn).parameters["antialiasing"].default is None, fn
    assert rasterizer.get_antialiasing() is False


def test_flag_reaches_the_config_and_a_stale_library_is_refused(capi, monkeypatch):
    from pf3plat_b200 import rasterizer
    from pf3plat_b200.rasterizer import BatchSettings, _make_config
    bs = BatchSettings(image_height=16, image_width=16, viewmatrix=torch.eye(4)[None], projmatrix=torch.eye(4)[None],
                       campos=torch.zeros(1, 3), bg=torch.zeros(1, 3), sh_degree=0)
    assert _make_config(bs, 1, 4, 0, []).flags & capi.GS_FLAG_ANTIALIAS == 0
    assert _make_config(bs._replace(antialiasing=True), 1, 4, 0, []).flags & capi.GS_FLAG_ANTIALIAS
    try:
        rasterizer.set_antialiasing(True)
        assert rasterizer.get_antialiasing() is True
        assert _make_config(bs, 1, 4, 0, []).flags & capi.GS_FLAG_ANTIALIAS
        assert _make_config(bs._replace(antialiasing=False), 1, 4, 0, []).flags & capi.GS_FLAG_ANTIALIAS == 0
        # the setting is resolved once, in the forward: its backward keeps it
        assert rasterizer._resolve_degree(bs).antialiasing is True
    finally:
        rasterizer.set_antialiasing(False)

    class Stale:   # a library of the same ABI version that predates the flag
        def gs_supported_flags(self):
            return capi.GS_FLAG_DEPTH | capi.GS_FLAG_PREFILTERED | capi.GS_FLAG_DETERMINISTIC

    monkeypatch.setattr(capi, "_lib", Stale())
    with pytest.raises(RuntimeError, match="anti-aliasing"):
        rasterizer.set_antialiasing(True)
    assert rasterizer.get_antialiasing() is False
    with pytest.raises(RuntimeError, match="anti-aliasing"):
        _make_config(bs._replace(antialiasing=True), 1, 4, 0, [])
    _make_config(bs, 1, 4, 0, [])   # without the flag nothing asks
