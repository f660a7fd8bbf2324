"""CPU checks of the degree-4 SH basis and of the degree-4 oracle (tests/sh4_oracle.py) the GPU tests compare against."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import torch_oracle
from pf3plat_b200.rasterizer import BatchSettings
from pf3plat_b200.sh_rotation import real_sh_basis
from pf3plat_b200.synthetic import make_scene, make_target
from tests.batch_oracle import batch_view_settings, oracle_batch, scene_batch_args
from tests.sh4_oracle import SH_C4, ShOracleBatch, sh_basis, with_band4
from tests.util import simple_settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")

BAND4_CONSTANTS = [2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892,
                   0.10578554691520431, -0.6690465435572892, 0.47308734787878004, -1.7701307697799304,
                   0.6258357354491761]


def _sphere_quadrature(nt=40, nphi=80):
    ct, wt = np.polynomial.legendre.leggauss(nt)
    phi = (np.arange(nphi) + 0.5) * 2 * np.pi / nphi
    st = np.sqrt(1 - ct * ct)
    d = np.stack([st[:, None] * np.cos(phi)[None], st[:, None] * np.sin(phi)[None], np.repeat(ct[:, None], nphi, 1)], -1)
    w = np.repeat(wt[:, None], nphi, 1) * (2 * np.pi / nphi)
    return d.reshape(-1, 3), w.reshape(-1)


def _unit(n, seed=0):
    u = np.random.default_rng(seed).standard_normal((n, 3))
    return u / np.linalg.norm(u, axis=-1, keepdims=True)


def test_basis_is_orthonormal_on_the_sphere():
    d, w = _sphere_quadrature()
    B = sh_basis(d, 4)
    gram = (B * w[:, None]).T @ B
    assert np.abs(gram - np.eye(25)).max() < 1e-12


def test_bands_0_to_3_are_the_oracles():
    u = _unit(500)
    B = sh_basis(u, 4)
    ut = torch.as_tensor(u)
    for k in range(16):
        shs = torch.zeros(500, 16, 3, dtype=torch.float64)
        shs[:, k, :] = 0.1
        rgb = torch_oracle._sh_rgb(3, shs, ut)          # 0.1 * Y_k + 0.5, never clamped at this scale
        assert np.abs((rgb[:, 0].numpy() - 0.5) / 0.1 - B[:, k]).max() < 1e-12, k


def test_band4_spans_real_sh_basis_through_an_orthogonal_map():
    u = _unit(400, seed=1)
    B4 = sh_basis(u, 4)[:, 16:25]
    R4 = real_sh_basis(4, torch.as_tensor(u)).numpy()
    Q, *_ = np.linalg.lstsq(R4, B4, rcond=None)
    assert np.abs(R4 @ Q - B4).max() < 1e-12
    assert np.abs(Q.T @ Q - np.eye(9)).max() < 1e-12


def test_band4_constants_are_pinned():
    assert SH_C4 == BAND4_CONSTANTS
    src = open(os.path.join(ROOT, "pf3plat_b200", "csrc", "gs_common.cuh")).read()
    for k, c in enumerate(BAND4_CONSTANTS):
        m = re.search(rf"#define GS_SH_C4_{k} \(?(-?[0-9.]+)f\)?", src)
        assert m and float(m.group(1)) == c, k


def _batch(scene, deg_scene=None, device="cpu"):
    cams, ins = scene_batch_args([scene], device=device)
    bs = BatchSettings(image_height=scene.image_shape[0], image_width=scene.image_shape[1], sh_degree=4, **cams)
    return bs, ins


def test_degree3_reproduces_the_committed_golden():
    z = np.load(os.path.join(G, "scene_sh_2k.npz"))
    views, h, w = int(z["views"]), int(z["h"]), int(z["w"])
    sc = make_scene(int(z["P"]), views, h, w, seed=int(z["seed"]))
    bs, ins = _batch(sc)
    orc = ShOracleBatch(bs, ins["means3D"], ins["opacities"], ins["shs"], deg=3, cov3D_precomp=ins["cov3D_precomp"],
                        dtype=np.float32)
    target = make_target(views, h, w).numpy()
    dL = (2 * (orc.color - target) / target.size).astype(np.float32)
    g = orc.backward(dL)
    s = orc.s
    for v in range(views):
        assert np.array_equal(orc.radii[v], z[f"radii{v}"])
        assert np.abs(orc.color[v] - z[f"color{v}"]).max() < 1e-5
    # the golden holds each view's gradient w.r.t. that view's scaled inputs: compare the sum over views
    gm = sum(z[f"g_means{v}"] * s[v] for v in range(views))
    assert np.abs(g["means3D"][0] - gm).max() <= 1e-4 * np.abs(gm).max()
    go = sum(z[f"g_opac{v}"][:, 0] for v in range(views))
    assert np.abs(g["opacities"][0] - go).max() <= 1e-5 * np.abs(go).max()


def test_degree3_composition_equals_the_c_oracle_in_fp64():
    sc = make_scene(300, 2, 32, 48, seed=3)
    bs, ins = _batch(sc)
    a = ShOracleBatch(bs, ins["means3D"], ins["opacities"], ins["shs"], deg=3, cov3D_precomp=ins["cov3D_precomp"])
    bs3 = bs._replace(sh_degree=3)
    b = oracle_batch(bs3, ins["means3D"], ins["opacities"], shs=ins["shs"], cov3D_precomp=ins["cov3D_precomp"],
                     dtype=np.float64)
    assert np.abs(a.color - b.color).max() < 1e-12
    dL = make_target(2, 32, 48).numpy() - 0.5
    ga, gb = a.backward(dL), b.backward(dL)
    for k in ("means3D", "opacities", "cov3D_precomp"):
        assert np.abs(ga[k] - gb[k]).max() <= 1e-10 * (np.abs(gb[k]).max() + 1e-30), k
    assert np.abs(ga["shs"][..., :16, :] - gb["shs"][..., :16, :]).max() <= 1e-10 * np.abs(gb["shs"]).max()
    assert not ga["shs"][..., 16:, :].any()


def _torch_restatement(bs, ins, M=25):
    """Single view: the SH colour through band 4 in torch, rendered by oracle/torch_oracle.py; gradients by autograd."""
    st = batch_view_settings(bs, 0, M)
    s = float(np.float32(bs.view_scale[0]))
    means = ins["means3D"][0].double().clone().requires_grad_(True)
    shs = ins["shs"][0].double().clone().requires_grad_(True)
    opac = ins["opacities"][0].double().clone().requires_grad_(True)
    cov = ins["cov3D_precomp"][0].double().clone().requires_grad_(True)
    m = means * s
    d = m - torch.as_tensor(st.campos, dtype=torch.float64)
    u = d / d.norm(dim=-1, keepdim=True)
    rgb = torch.clamp_min(torch.einsum("pk,pkc->pc", sh_basis(u, 4), shs) + 0.5, 0.0)
    color, _ = torch_oracle.render(st, m, opac, colors_precomp=rgb, cov3D_precomp=cov * (s * s))
    return color, (means, shs, opac, cov)


@pytest.fixture(scope="module")
def small_band4():
    sc = with_band4(make_scene(120, 1, 32, 32, seed=5))
    bs, ins = _batch(sc)
    orc = ShOracleBatch(bs, ins["means3D"], ins["opacities"], ins["shs"], deg=4, cov3D_precomp=ins["cov3D_precomp"])
    return sc, bs, ins, orc


def test_degree4_oracle_matches_autograd_restatement(small_band4):
    sc, bs, ins, orc = small_band4
    color, leaves = _torch_restatement(bs, ins)
    assert np.abs(color.detach().numpy() - orc.color[0]).max() < 1e-9
    Wt = torch.as_tensor(make_target(1, 32, 32).numpy()[0] - 0.5, dtype=torch.float64)
    (color * Wt).sum().backward()
    g = orc.backward(Wt.numpy()[None])
    means, shs, opac, cov = leaves
    for name, t, ref in (("means3D", means, g["means3D"][0]), ("opacities", opac, g["opacities"][0]),
                         ("cov3D", cov, g["cov3D_precomp"][0]), ("shs", shs, g["shs"][0])):
        a = t.grad.numpy()
        # (the tolerance of tests/test_oracle_gradients.py: relative to the largest element)
        assert np.abs(a - ref).max() <= 1e-5 * (np.abs(ref).max() + 1e-30), name
    assert np.abs(g["shs"][0, :, 16:25]).max() > 1e-3       # band 4 receives a gradient


def test_degree4_finite_differences(small_band4):
    sc, bs, ins, orc = small_band4
    Wt = make_target(1, 32, 32).numpy() - 0.5
    g = orc.backward(Wt)

    def loss(means=None, shs=None):
        o = ShOracleBatch(bs, ins["means3D"] if means is None else means, ins["opacities"],
                          ins["shs"] if shs is None else shs, deg=4, cov3D_precomp=ins["cov3D_precomp"])
        return float((o.color * Wt).sum())

    aff = orc.affected()[0]
    # the visible, non-fragile Gaussians with the largest colour gradient
    order = np.argsort(-np.abs(g["shs"][0, :, 0, 0]))
    pick = [p for p in order if not aff[p]][:4]
    assert len(pick) == 4
    h = 1e-6
    for p in pick:
        for k, c in ((16, 0), (20, 1), (24, 2)):
            sp, sm = ins["shs"].double().clone(), ins["shs"].double().clone()
            sp[0, p, k, c] += h
            sm[0, p, k, c] -= h
            fd = (loss(shs=sp) - loss(shs=sm)) / (2 * h)
            assert abs(fd - g["shs"][0, p, k, c]) <= 1e-6 * abs(fd) + 1e-9, (p, k, c, fd, g["shs"][0, p, k, c])
        for a in range(3):
            mp, mm = ins["means3D"].double().clone(), ins["means3D"].double().clone()
            mp[0, p, a] += h
            mm[0, p, a] -= h
            fd = (loss(means=mp) - loss(means=mm)) / (2 * h)
            assert abs(fd - g["means3D"][0, p, a]) <= 1e-4 * abs(fd) + 1e-7, (p, a, fd, g["means3D"][0, p, a])


@pytest.mark.parametrize("k", [18, 19, 20])
def test_closed_form_centre_pixel(k):
    """One Gaussian projecting exactly onto pixel (32, 32) of an identity camera, colour from sh[0] and one band-4
    coefficient: the centre pixel is alpha * (C0 sh_0 + Y_k(dir) sh_k + 0.5) (black background, G = 1 there)."""
    st = simple_settings(64, 64, tanfov=0.5, sh_degree=4)
    z = 5.0
    mean = np.array([[z / 128, z / 128, z]])
    x, y, zz_ = mean[0] / np.linalg.norm(mean[0])
    poly = {18: 0.9461746957575601 * x * y * (7 * zz_ * zz_ - 1),
            20: 0.10578554691520431 * (zz_ * zz_ * (35 * zz_ * zz_ - 30) + 3),
            19: -0.6690465435572892 * y * zz_ * (7 * zz_ * zz_ - 3)}[k]
    shs = np.zeros((1, 1, 25, 3))
    shs[0, 0, 0] = [0.3, -0.2, 0.1]
    shs[0, 0, k] = [0.4, 0.25, -0.3]
    f = lambda a: torch.as_tensor(np.asarray(a, np.float32))[None]
    bs = BatchSettings(image_height=64, image_width=64, viewmatrix=f(st.viewmatrix), projmatrix=f(st.projmatrix),
                       campos=f(st.campos), bg=f(st.bg), sh_degree=4, tanfovx=0.5, tanfovy=0.5)
    cov = np.array([[[0.01, 0, 0, 0.01, 0, 0.01]]])
    orc = ShOracleBatch(bs, mean[None].astype(np.float32), np.array([[0.6]]), shs, deg=4, cov3D_precomp=cov)
    expect = 0.6 * np.maximum(0.28209479177387814 * shs[0, 0, 0] + poly * shs[0, 0, k] + 0.5, 0.0)
    assert np.abs(orc.color[0, :, 32, 32] - expect).max() < 1e-6
    if k != 20:
        assert abs(poly) > 1e-4   # the band-4 term is really there
