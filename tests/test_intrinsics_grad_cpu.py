"""CPU tests of the intrinsics gradient: the oracle of tests/intrinsics_oracle.py against central finite differences in
tanfov of the fp64 forward it differentiates (Gaussians beyond the guard band included, with anti-aliasing, SH degree 4,
the four depth modes and alpha); make_view_batch's glue against the reference's own (tests/golden/intrinsics_glue.npz);
and the C ABI's declaration of gs_backward_cam_tanfov against its ctypes mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from tests.camera_oracle import camera_oracle, view_loss
from tests.intrinsics_oracle import clamped_pairs, intrinsics_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "intrinsics_glue.npz")


def scene(P=24, hw=(24, 32), seed=0, use_sh=True, M=16, n_edge=4):
    """One scene, two views with unequal tanfov per axis and per view.  The first P Gaussians lie well inside the frustum;
    n_edge large ones lie beyond the guard band (|t.x / t.z| or |t.y / t.z| > 1.3 tanfov) with footprints that still
    reach into the frame, so the clamp branch feeds the loss.  The seeds the tests use keep every splat farther than
    the finite-difference step from a tile edge and from the 1/255 threshold."""
    from pf3plat_b200.rasterizer import BatchSettings
    g = torch.Generator().manual_seed(seed)
    V = 2
    tan = torch.tensor([[0.6, 0.45], [0.5, 0.55]], dtype=torch.float64)
    inner = torch.cat([torch.rand(1, P, 2, generator=g) * 1.2 - 0.6, 4 + torch.rand(1, P, 1, generator=g) * 2], -1)
    s = 0.05 + 0.1 * torch.rand(1, P, 3, generator=g)
    # beyond the band: x / z (or y / z) of 0.85..0.95 at z 4..5, alternately left, right, top and bottom
    k = torch.arange(n_edge)
    r = 0.85 + 0.1 * torch.rand(n_edge, generator=g)
    z = 4 + torch.rand(n_edge, generator=g)
    sgn = torch.where(k % 2 == 0, 1.0, -1.0)
    ex = torch.where(k % 4 < 2, sgn * r * z, 0.1 * torch.randn(n_edge, generator=g))
    ey = torch.where(k % 4 < 2, 0.1 * torch.randn(n_edge, generator=g), sgn * r * z)
    edge = torch.stack([ex, ey, z], -1)[None]
    es = 0.6 + 0.3 * torch.rand(1, n_edge, 3, generator=g)
    means = torch.cat([inner, edge], 1)
    sc = torch.cat([s, es], 1)
    Pt = P + n_edge
    cov = torch.zeros(1, Pt, 6)
    cov[..., 0], cov[..., 3], cov[..., 5] = sc[..., 0] ** 2, sc[..., 1] ** 2, sc[..., 2] ** 2
    ins = {"means3D": means.double(), "opacities": (0.3 + 0.4 * torch.rand(1, Pt, generator=g)).double(),
           "cov3D_precomp": cov.double()}
    if use_sh:
        ins["shs"] = (0.3 * torch.randn(1, Pt, M, 3, generator=g)).double()
    else:
        ins["colors_precomp"] = torch.rand(V, Pt, 3, generator=g).double()
    view = torch.eye(4, dtype=torch.float64).repeat(V, 1, 1)
    view[1, 3, 0], view[1, 3, 1] = 0.2, -0.1              # translation row of the transposed matrix
    proj = torch.zeros(V, 4, 4, dtype=torch.float64)
    n, f = 0.5, 50.0
    for v in range(V):
        Pm = torch.zeros(4, 4, dtype=torch.float64)
        Pm[0, 0], Pm[1, 1], Pm[2, 2], Pm[2, 3], Pm[3, 2] = 1 / tan[v, 0], 1 / tan[v, 1], f / (f - n), 1.0, -f * n / (f - n)
        proj[v] = view[v] @ Pm
    campos = -view[:, 3, :3]
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=view, projmatrix=proj, campos=campos,
                       bg=torch.tensor([[0.1, 0.2, 0.3]] * V, dtype=torch.float64), sh_degree=4 if M >= 25 else 3,
                       tanfov=tan, view_scale=torch.tensor([1.0, 0.8]), with_depth=True,
                       sh_eval_max_degree=4 if M >= 25 else 3)
    return bs, ins


CASES = {
    "sh3_depth": dict(),
    "colors_alpha": dict(use_sh=False, alpha=True),
    "aa_disparity": dict(kw={"antialiasing": True, "depth_mode": "disparity"}),
    "sh4_relative": dict(M=25, kw={"depth_mode": "relative_disparity", "near_far": np.array([[0.5, 50.0], [0.6, 40.0]])}),
    "aa_log_alpha": dict(alpha=True, kw={"antialiasing": True, "depth_mode": "log",
                                         "near_far": np.array([[0.5, 50.0], [0.6, 40.0]])}),
}


def _case(case):
    c = CASES[case]
    bs, ins = scene(use_sh=c.get("use_sh", True), M=c.get("M", 16))
    V, H, W = 2, bs.image_height, bs.image_width
    rng = np.random.default_rng(1)
    dL = rng.standard_normal((V, 3, H, W))
    w = rng.standard_normal((V, H, W))
    dA = rng.standard_normal((V, H, W)) if c.get("alpha") else None
    return bs, ins, dL, w, dA, c.get("kw", {})


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_finite_differences_in_tanfov(case):
    bs, ins, dL, w, dA, kw = _case(case)
    assert all(clamped_pairs(bs, ins, v) >= 4 for v in range(2))
    got = intrinsics_oracle(bs, ins, dL, w, dA, **kw)[3]
    scale = np.abs(got).max() + 1e-12
    assert scale > 1e-3
    h = 1e-6
    for v in range(2):
        for e in range(2):
            out = []
            for sgn in (1, -1):
                t = bs.tanfov.clone()
                t[v, e] += sgn * h
                with torch.no_grad():
                    out.append(float(view_loss(bs._replace(tanfov=t), ins, v, dL, w, dA, **kw)[0]))
            fd = (out[0] - out[1]) / (2 * h)
            assert abs(fd - got[v, e]) <= 1e-5 * scale + 1e-4 * abs(got[v, e]), (case, v, e, fd, got[v, e])


def test_clamp_term_is_what_the_composition_adds():
    """Beyond the guard band the clamp's own term matters: without it (autograd of the oracle as it stands) the
    gradient of the clamped Gaussians differs from the finite difference, with it the two agree (above)."""
    import tests.intrinsics_oracle as io
    bs, ins, dL, w, dA, kw = _case("sh3_depth")
    full = intrinsics_oracle(bs, ins, dL, w, dA, **kw)[3]
    orig = io.clamp_compensated_sigma
    try:
        io.clamp_compensated_sigma = lambda st, view, tan, means, Sig: Sig
        plain = intrinsics_oracle(bs, ins, dL, w, dA, **kw)[3]
    finally:
        io.clamp_compensated_sigma = orig
    assert np.abs(full - plain).max() > 1e-3 * np.abs(full).max()


@pytest.mark.parametrize("case", ["sh3_depth", "aa_log_alpha"])
def test_camera_leaves_are_the_camera_oracles(case):
    """tanfov as a fourth leaf leaves the forward and the other three gradients as tests/camera_oracle.py gives them."""
    bs, ins, dL, w, dA, kw = _case(case)
    a = camera_oracle(bs, ins, dL, w, dA, **kw)
    b = intrinsics_oracle(bs, ins, dL, w, dA, **kw)
    for x, y in zip(a, b[:3]):
        np.testing.assert_allclose(y, x, rtol=1e-12, atol=1e-12 * (np.abs(x).max() + 1e-30))


# ---------------------------------------------------------------------------------------------------------
# the glue: intrinsics -> tanfov, P, full projection (pf3plat_b200.cameras on CPU tensors) against the reference's own
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["si", "raw"])
def test_glue_matches_the_reference_glue_and_its_vjps(tag):
    from pf3plat_b200.cameras import get_fov, get_projection_matrix, make_view_batch
    z = np.load(GOLDEN)
    t = lambda k: torch.from_numpy(z[k])
    ext, near, far = t("extrinsics"), t("near"), t("far")
    K = t("intrinsics").clone().requires_grad_(True)
    vb = make_view_batch(ext, K, near, far, scale_invariant=tag == "si", camera_gradients=True)
    fov_x, fov_y = get_fov(K).unbind(-1)
    nr, fr = (near * (1 / near), far * (1 / near)) if tag == "si" else (near, far)
    P = get_projection_matrix(nr, fr, fov_x, fov_y)
    for k, got in (("tanfov", vb.tanfov), ("P", P), ("full", vb.projmatrix)):
        assert got.dtype == torch.float64
        np.testing.assert_allclose(got.detach().numpy(), z[f"{tag}_{k}"], rtol=0, atol=1e-10, err_msg=k)
        vjp = torch.autograd.grad((got * t(f"cot_{k}")).sum(), K, retain_graph=True)[0].numpy()
        np.testing.assert_allclose(vjp, z[f"{tag}_vjp_{k}"], rtol=0, atol=1e-10, err_msg=k)
        assert np.abs(vjp).max() > 1e-3
    # the principal point and the skew change the fov: their entries of the tanfov VJP are not zero
    g = z[f"{tag}_vjp_tanfov"]
    assert (np.abs(g[:, 0, 2]) > 1e-6).all() and (np.abs(g[:, 1, 2]) > 1e-6).all() and (np.abs(g[:, 0, 1]) > 1e-6).all()


# ---------------------------------------------------------------------------------------------------------
# the C ABI
# ---------------------------------------------------------------------------------------------------------
def test_header_declares_the_entry_as_the_binding_calls_it(tmp_path):
    """gs_backward_cam_tanfov: gs_backward_cam's arguments, then float *dL_dtanfov, then the stream -- in the header
    (checked by compiling a call with those types) and in _capi's prototype.  GsCameraGrads keeps its layout."""
    from pf3plat_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert "GS_API int gs_backward_cam_tanfov(" in hdr
    prog = tmp_path / "tan.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\n'
                    'int (*fn)(GsContext *, const GsConfig *, const GsInputs *, const GsSaved *, const GsOutGrads *,'
                    ' const GsAlpha *, const GsInGrads *, const GsCameraGrads *, float *, void *) = gs_backward_cam_tanfov;\n'
                    'int main(void){printf("%zu %zu\\n", sizeof(GsCameraGrads), offsetof(GsCameraGrads, dL_dcampos));'
                    'return 0;}\n')
    subprocess.run(["gcc", "-Werror", "-Wincompatible-pointer-types", "-I", os.path.join(ROOT, "include"), "-c",
                    str(prog), "-o", str(tmp_path / "tan.o")], check=True)
    res, args = _capi.SYMBOLS["gs_backward_cam_tanfov"]
    cam_res, cam_args = _capi.SYMBOLS["gs_backward_cam"]
    assert res is cam_res and args[:8] == cam_args[:8] and args[8:] == [ctypes.c_void_p, ctypes.c_void_p]
    assert ctypes.sizeof(_capi.GsCameraGrads) == 3 * ctypes.sizeof(ctypes.c_void_p)


def test_a_library_without_the_entry_is_refused(tmp_path, monkeypatch):
    """The binding loads gs_backward_cam_tanfov with the other symbols: a library of the same ABI version that predates it
    fails to load, rather than leaving the intrinsics without their gradient silently."""
    from pf3plat_b200 import _capi
    names = [n for n in _capi.SYMBOLS if n != "gs_backward_cam_tanfov"]
    src = tmp_path / "old.c"
    src.write_text("".join(f"int {n}(void) {{ return {_capi.ABI_VERSION if n == 'gs_abi_version' else 0}; }}\n"
                           for n in names))
    so = tmp_path / "libold.so"
    subprocess.run(["gcc", "-shared", "-fPIC", str(src), "-o", str(so)], check=True)
    monkeypatch.setattr(_capi, "LIB_PATH", str(so))
    monkeypatch.setattr(_capi, "_lib", None)
    with pytest.raises(AttributeError, match="gs_backward_cam_tanfov"):
        _capi.lib()

