"""CPU tests of the camera gradient: the oracle of tests/camera_oracle.py against central finite differences of the fp64
forward it differentiates (colour, depth in every mode, alpha, anti-aliasing), the C ABI's declarations, and the Python
settings."""
import inspect
import os
import subprocess

import numpy as np
import pytest
import torch

from tests.camera_oracle import camera_oracle, view_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _scene(P=24, hw=(24, 32), seed=0, use_sh=True):
    """One scene, two views, Gaussians well inside the frustum.  The derivative jumps where a splat crosses a tile edge or
    the 1/255 threshold; the seeds the tests use were checked, entry by entry, to keep every such crossing farther than
    the finite-difference step (seed 3, for one, does not: with anti-aliasing one splat of view 0 sits on a threshold)."""
    from pf3plat_b200.rasterizer import BatchSettings
    g = torch.Generator().manual_seed(seed)
    V = 2
    means = torch.cat([torch.rand(1, P, 2, generator=g) * 1.6 - 0.8, 4 + torch.rand(1, P, 1, generator=g) * 2], -1)
    cov = torch.zeros(1, P, 6)
    s = 0.05 + 0.1 * torch.rand(1, P, 3, generator=g)
    cov[..., 0], cov[..., 3], cov[..., 5] = s[..., 0] ** 2, s[..., 1] ** 2, s[..., 2] ** 2
    ins = {"means3D": means.double(), "opacities": (0.3 + 0.4 * torch.rand(1, P, generator=g)).double(),
           "cov3D_precomp": cov.double()}
    if use_sh:
        ins["shs"] = (0.3 * torch.randn(1, P, 16, 3, generator=g)).double()
    else:
        ins["colors_precomp"] = torch.rand(V, P, 3, generator=g).double()
    view = torch.eye(4, dtype=torch.float64).repeat(V, 1, 1)
    view[1, 3, 0], view[1, 3, 1] = 0.2, -0.1              # translation row of the transposed matrix
    tan = 0.6
    P_ = torch.zeros(4, 4, dtype=torch.float64)
    n, f = 0.5, 50.0
    P_[0, 0], P_[1, 1], P_[2, 2], P_[2, 3], P_[3, 2] = 1 / tan, 1 / tan, f / (f - n), 1.0, -f * n / (f - n)
    proj = view @ P_
    campos = -view[:, 3, :3]
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=view, projmatrix=proj, campos=campos,
                       bg=torch.tensor([[0.1, 0.2, 0.3]] * V, dtype=torch.float64), sh_degree=3, tanfovx=tan,
                       tanfovy=tan, view_scale=torch.tensor([1.0, 0.8]), with_depth=True)
    return bs, ins


def _fd(bs, ins, dL, w, dA, kw, which, idx, h=1e-6):
    """Central difference of view v's fp64 loss in bs.<which>[v].flat[e]."""
    v, e = idx
    out = []
    for sgn in (1, -1):
        t = getattr(bs, which).clone()
        t.reshape(t.shape[0], -1)[v, e] += sgn * h
        with torch.no_grad():
            out.append(float(view_loss(bs._replace(**{which: t}), ins, v, dL, w, dA, **kw)[0]))
    return (out[0] - out[1]) / (2 * h)


@pytest.mark.parametrize("case", ["sh_depth", "colors_alpha", "aa_disparity", "log_relative"])
def test_oracle_matches_finite_differences(case):
    use_sh = case != "colors_alpha"
    bs, ins = _scene(use_sh=use_sh, seed=0)
    V, H, W = 2, bs.image_height, bs.image_width
    rng = np.random.default_rng(1)
    dL = rng.standard_normal((V, 3, H, W))
    w = rng.standard_normal((V, H, W))
    dA = rng.standard_normal((V, H, W)) if case == "colors_alpha" else None
    kw = {}
    if case == "aa_disparity":
        kw = {"antialiasing": True, "depth_mode": "disparity"}
    if case == "log_relative":
        kw = {"depth_mode": "relative_disparity", "near_far": np.array([[0.5, 50.0], [0.6, 40.0]])}
    got = camera_oracle(bs, ins, dL, w, dA, **kw)
    for j, which in enumerate(("viewmatrix", "projmatrix", "campos")):
        n = got[j].shape[1]
        for v in range(V):
            for e in range(n):   # every entry, the ones that feed nothing included (both sides must be 0 there)
                fd = _fd(bs, ins, dL, w, dA, kw, which, (v, e))
                ref = got[j][v, e]
                scale = np.abs(got[j]).max() + 1e-12
                assert abs(fd - ref) <= 1e-5 * scale + 1e-4 * abs(ref), (case, which, v, e, fd, ref)


def test_header_declares_the_entry_and_the_struct_layout(tmp_path):
    hdr = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert "GS_API int gs_backward_cam(" in hdr
    prog = tmp_path / "cam.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %zu %zu\\n", sizeof(GsCameraGrads), offsetof(GsCameraGrads, dL_dviewmatrix),'
                    'offsetof(GsCameraGrads, dL_dprojmatrix), offsetof(GsCameraGrads, dL_dcampos));return 0;}')
    exe = tmp_path / "cam"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    sizes = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    from pf3plat_b200._capi import GsCameraGrads
    assert sizes == [ctypes_sizeof(GsCameraGrads), GsCameraGrads.dL_dviewmatrix.offset, GsCameraGrads.dL_dprojmatrix.offset,
                     GsCameraGrads.dL_dcampos.offset]


def ctypes_sizeof(t):
    import ctypes
    return ctypes.sizeof(t)


def test_settings_default_off_and_entry_points():
    from pf3plat_b200 import rasterizer
    from pf3plat_b200.cameras import make_view_batch
    from pf3plat_b200.rasterizer import BatchSettings, GaussianRasterizer
    from pf3plat_b200.render import decoder_forward, render_views
    assert rasterizer.get_camera_gradients() is False
    assert BatchSettings._field_defaults["camera_gradients"] is None
    for fn in (GaussianRasterizer.forward, render_views, decoder_forward, make_view_batch):
        assert inspect.signature(fn).parameters["camera_gradients"].default is None, fn
    rasterizer.set_camera_gradients(True)
    try:
        assert rasterizer.get_camera_gradients() is True
    finally:
        rasterizer.set_camera_gradients(False)


def test_a_library_without_the_entry_is_refused(tmp_path, monkeypatch):
    """The binding loads gs_backward_cam with the other symbols: a library of the same ABI version that predates it fails
    to load, rather than leaving the camera gradient out silently."""
    from pf3plat_b200 import _capi
    names = [n for n in _capi.SYMBOLS if n != "gs_backward_cam"]
    src = tmp_path / "old.c"
    src.write_text("".join(f"int {n}(void) {{ return {_capi.ABI_VERSION if n == 'gs_abi_version' else 0}; }}\n"
                           for n in names))
    so = tmp_path / "libold.so"
    subprocess.run(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)], check=True)
    monkeypatch.setattr(_capi, "LIB_PATH", str(so))
    monkeypatch.setattr(_capi, "_lib", None)
    with pytest.raises(AttributeError, match="gs_backward_cam"):
        _capi.lib()
