"""CPU checks of the accumulated-opacity output: the fp64 oracle composition of tests/alpha_oracle.py against an autograd
restatement of 1 - prod_i (1 - alpha_i) (oracle/torch_oracle.py, whose background term is T_final = that product) and
against finite differences of its own forward; and the C-ABI pieces -- exported entry points, the GsAlpha layout, the
requests the library refuses, the unchanged ABI version and output structs."""
import ctypes
import dataclasses
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import torch_oracle
from pf3plat_b200.synthetic import make_scene
from tests.alpha_oracle import AlphaOracle
from tests.batch_oracle import batch_view_settings, scene_batch_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _single_view(geometry, seed=5, P=400, hw=(32, 48)):
    from pf3plat_b200.rasterizer import BatchSettings
    sc = make_scene(P, 1, *hw, seed=seed)
    cams, ins = scene_batch_args([sc])
    keep = ("means3D", "opacities", "shs") + (("cov3D_precomp",) if geometry == "cov3D" else ("scales", "rotations"))
    ins = {k: ins[k].double() for k in keep}
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=cams["viewmatrix"], projmatrix=cams["projmatrix"],
                       campos=cams["campos"], bg=cams["bg"], sh_degree=3, tanfov=cams["tanfov"])
    return bs, ins


def _torch_alpha(bs, ins):
    """alpha = 1 - T_final by autograd: colours 0 on a white background render exactly T_final = prod_i (1 - alpha_i)."""
    st = dataclasses.replace(batch_view_settings(bs, 0, 0), bg=np.ones(3))
    tk = {k: v[0].clone().requires_grad_(True) for k, v in ins.items() if k != "shs"}
    P = tk["means3D"].shape[0]
    color, _ = torch_oracle.render(st, colors_precomp=torch.zeros(P, 3, dtype=torch.float64), **tk)
    return 1.0 - color[0], tk


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_composition_matches_the_autograd_restatement(geometry):
    bs, ins = _single_view(geometry)
    orc = AlphaOracle(bs, ins)
    alpha_t, leaves = _torch_alpha(bs, ins)
    a = alpha_t.detach().numpy()
    covered = float((orc.alpha > 0).mean())
    print(f"[regime] {geometry}: alpha {orc.alpha.min():.3f}..{orc.alpha.max():.3f}, covered pixels {covered:.2f}, "
          f"max |composition - autograd| {np.abs(a - orc.alpha[0]).max():.2e}")
    assert 0.2 < covered < 1.0 and orc.alpha.max() > 0.9
    np.testing.assert_allclose(orc.alpha[0], a, rtol=0, atol=1e-12)
    assert np.all(orc.alpha[orc.final_T == 1.0] == 0.0)   # no contributor: exactly 0
    w = np.random.default_rng(1).standard_normal(a.shape)
    (alpha_t * torch.as_tensor(w)).sum().backward()
    g = orc.alpha_grads(w[None])
    assert g["colors_precomp"] is None
    for k, t in leaves.items():
        want = t.grad.numpy()
        got = g[k][0].reshape(want.shape)
        scale = np.abs(want).max()
        err = np.abs(got - want).max()
        print(f"[parity] {geometry} dL/d{k}: max |composition - autograd| {err:.2e} of {scale:.2e}")
        assert scale > 0 and err <= 1e-5 * scale, k


def test_composition_matches_finite_differences():
    """Directional derivatives of <w, alpha> in fp64 along random directions of the opacities and of the means of
    Gaussians that sit at no fragile decision."""
    from tests.batch_oracle import oracle_batch
    bs, ins = _single_view("cov3D", seed=9, P=300)
    orc = AlphaOracle(bs, ins)
    w = np.random.default_rng(2).standard_normal(orc.alpha.shape)
    g = orc.alpha_grads(w)
    safe = ~orc.ob_alpha.affected()[0]
    rng = np.random.default_rng(3)
    geo = {k: v for k, v in ins.items() if k != "shs"}
    P = geo["means3D"].shape[1]
    bs0 = bs._replace(bg=torch.zeros(1, 3, dtype=torch.float64))

    def loss(inputs):
        ob = oracle_batch(bs0, colors_precomp=np.ones((1, P, 3)), dtype=np.float64, **inputs)
        return float((ob.color[:, 0] * w).sum())

    for k, h in (("opacities", 1e-7), ("means3D", 1e-7)):
        d = rng.standard_normal(geo[k].shape) * safe.reshape((1, P) + (1,) * (geo[k].dim() - 2))
        plus = {**geo, k: geo[k] + h * torch.as_tensor(d)}
        minus = {**geo, k: geo[k] - h * torch.as_tensor(d)}
        fd = (loss(plus) - loss(minus)) / (2 * h)
        an = float((g[k].reshape(d.shape) * d).sum())
        print(f"[parity] finite differences dL/d{k}: analytic {an:.6e}, central difference {fd:.6e}")
        assert abs(an) > 0 and abs(fd - an) <= 1e-5 * abs(an), k


# ---------------------------------------------------------------------------------------------------------------------
# the C ABI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_new_entry_points_are_exported_with_prototypes(capi):
    L = capi.lib()
    for name in ("gs_forward_ex", "gs_backward_ex", "gs_render_host_ex"):
        assert hasattr(L, name) and name in capi.SYMBOLS, name
    assert capi.ABI_VERSION == 5 and L.gs_abi_version() == 5


def test_struct_layouts_match_the_header(capi, tmp_path):
    prog = tmp_path / "alpha.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %zu %zu %zu %d\\n", sizeof(GsAlpha), offsetof(GsAlpha, alpha),'
                    'offsetof(GsAlpha, dL_dalpha), sizeof(GsOutputs), sizeof(GsOutGrads), GS_ABI_VERSION);return 0;}')
    exe = tmp_path / "alpha"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    A = capi.GsAlpha
    assert [ctypes.sizeof(A), A.alpha.offset, A.dL_dalpha.offset] == out[:3]
    # the output and incoming-gradient structs did not grow: alpha travels in GsAlpha
    assert out[3:5] == [3 * ctypes.sizeof(ctypes.c_void_p), 2 * ctypes.sizeof(ctypes.c_void_p)]
    assert [ctypes.sizeof(capi.GsOutputs), ctypes.sizeof(capi.GsOutGrads)] == out[3:5]
    assert out[5] == 5


def _request(capi):
    """A forward request that is valid in every respect but the alpha one (device pointers are never dereferenced)."""
    fake = 256
    cfg = capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = 16, 1, 1, 0, 0
    cfg.image_height, cfg.image_width, cfg.scale_modifier = 16, 16, 1.0
    cfg.viewmatrix = cfg.projmatrix = cfg.campos = cfg.bg = fake
    gin = capi.GsInputs(means3D=fake, opacities=fake, colors_precomp=fake, cov3D_precomp=fake)
    gout = capi.GsOutputs(color=fake, radii=fake)
    return cfg, gin, gout


@pytest.mark.parametrize("which", ["null struct", "null alpha"])
def test_forward_entries_refuse_a_request_without_an_alpha_buffer(capi, which):
    L = capi.lib()
    cfg, gin, gout = _request(capi)
    req = None if which == "null struct" else ctypes.byref(capi.GsAlpha(None, 256))
    fake_ctx = ctypes.c_void_p(256)
    saved = ctypes.c_void_p(1234)
    assert L.gs_forward_ex(fake_ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), req, ctypes.byref(saved),
                           None) == -1
    assert b"alpha" in L.gs_last_error() and not saved.value   # no handle is returned
    assert L.gs_render_host_ex(fake_ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), req, None) == -1
    assert b"alpha" in L.gs_last_error()


def test_backward_entry_refuses_null_arguments(capi):
    L = capi.lib()
    cfg, gin, _ = _request(capi)
    og = capi.GsOutGrads(256, None)
    ig = capi.GsInGrads()
    fake = ctypes.c_void_p(256)
    assert L.gs_backward_ex(fake, ctypes.byref(cfg), ctypes.byref(gin), fake, ctypes.byref(og), None, ctypes.byref(ig),
                            None) == -1
    assert b"null alpha" in L.gs_last_error()
    assert L.gs_backward_ex(None, None, None, None, None, ctypes.byref(capi.GsAlpha()), None, None) == -1
    assert b"null" in L.gs_last_error()


def test_batch_settings_append_with_alpha_last():
    from pf3plat_b200.rasterizer import BatchSettings, GaussianRasterizer
    assert BatchSettings._fields[-1] == "with_alpha" and BatchSettings._field_defaults["with_alpha"] is False
    import inspect
    p = inspect.signature(GaussianRasterizer.forward).parameters["return_alpha"]
    assert p.default is False
