"""The batched oracle (tests/batch_oracle.py), without a GPU: at one view of one scene it is the per-view oracle bit for
bit; its view-scale and scale-modifier chain rule and its per-scene sums agree with fp64 central finite differences of
the fp64 oracle."""
import numpy as np
import pytest
import torch

from pf3plat_b200.rasterizer import BatchSettings
from pf3plat_b200.synthetic import make_scene
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.util import oracle_view


def _settings(cams, hw, sh_degree=4, scale_modifier=1.0, with_depth=False):
    return BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=cams["viewmatrix"],
                         projmatrix=cams["projmatrix"], campos=cams["campos"], bg=cams["bg"], sh_degree=sh_degree,
                         tanfov=cams["tanfov"], view_scale=cams["view_scale"], scale_modifier=scale_modifier,
                         with_depth=with_depth)


@pytest.mark.parametrize("use_sh", [True, False])
def test_single_view_is_bit_identical_to_oracle_view(use_sh):
    sc = make_scene(2000, 3, 48, 64, seed=21)
    one = make_scene(2000, 1, 48, 64, seed=21, first_view=1, total_views=3)   # view 1 of the same scene on its own
    cams, ins = scene_batch_args([one], use_sh=use_sh)
    assert float(cams["view_scale"][0]) == 1.0
    colors = None if use_sh else sc.harmonics.permute(0, 2, 1)[:, 0, :].contiguous()[None]
    ob = oracle_batch(_settings(cams, (48, 64)), ins["means3D"], ins["opacities"], shs=ins.get("shs"),
                      colors_precomp=colors, cov3D_precomp=ins["cov3D_precomp"])
    ref = oracle_view(sc, 1, use_sh=use_sh)
    assert np.array_equal(ob.views[0].color, ref.color) and np.array_equal(ob.radii[0], ref.radii)
    rng = np.random.default_rng(0)
    dL = rng.standard_normal((1, 3, 48, 64)).astype(np.float32)
    g, gr = ob.backward(dL), ref.backward(dL[0])
    for name in ("means3D", "cov3D_precomp", "shs" if use_sh else "colors_precomp", "means2D"):
        assert np.array_equal(g[name][0], gr[name]), name
    assert np.array_equal(g["opacities"][0], gr["opacities"][:, 0])


def _fd_check(make_loss, base, g, rng, n=10, label=""):
    """Central differences of make_loss(perturbed base) at n random elements against g (same shape as base)."""
    flat_g = np.asarray(g, np.float64).reshape(-1)
    scale = np.abs(flat_g).max()
    assert scale > 0, label
    for i in rng.choice(base.size, size=n, replace=False):
        eps = 1e-6 * max(1.0, abs(base.reshape(-1)[i]))
        p, m = base.copy().reshape(-1), base.copy().reshape(-1)
        p[i] += eps
        m[i] -= eps
        fd = (make_loss(p.reshape(base.shape)) - make_loss(m.reshape(base.shape))) / (2 * eps)
        assert abs(fd - flat_g[i]) < 2e-4 * scale + 1e-9, (label, int(i), fd, flat_g[i])


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_view_scale_and_scale_modifier_chain_rule_matches_finite_differences(geometry):
    """S = 2 scenes x 2 views, view_scale 0.8 / 1.25 / 1.7 / 0.6, depth output on; scales + rotations with
    scale_modifier 0.7 and quaternions of norm != 1."""
    P, hw = 40, (32, 32)
    scenes = [make_scene(P, 2, *hw, seed=31 + k) for k in range(2)]
    near = [1.25, 0.8, 1 / 1.7, 1 / 0.6]
    cams, ins = scene_batch_args(scenes, near=near)
    assert np.allclose(cams["view_scale"].numpy(), [0.8, 1.25, 1.7, 0.6], rtol=1e-6)
    mod = 0.7 if geometry == "scalerot" else 1.0
    bs = _settings(cams, hw, scale_modifier=mod, with_depth=True)
    kw = {k: ins[k].double().numpy() for k in ("means3D", "opacities", "shs")}
    if geometry == "scalerot":
        kw["scales"] = ins["scales"].double().numpy() / mod
        kw["rotations"] = ins["rotations"].double().numpy() * np.linspace(0.6, 1.5, 2 * P).reshape(2, P, 1)
    else:
        kw["cov3D_precomp"] = ins["cov3D_precomp"].double().numpy()
    rng = np.random.default_rng(1)
    dL = rng.standard_normal((4, 3, *hw))
    dLd = rng.standard_normal((4, *hw)) * 1e-2

    def loss(**over):
        ob = oracle_batch(bs, dtype=np.float64, frag_rel=0, **{**kw, **over})
        return float((ob.color * dL).sum() + (ob.depth * dLd).sum())

    ob = oracle_batch(bs, dtype=np.float64, **kw)
    assert (ob.radii > 0).mean() > 0.5
    g = ob.backward(dL, dLd)
    names = ["means3D", "opacities"] + (["scales", "rotations"] if geometry == "scalerot" else ["cov3D_precomp"])
    for name in names:
        _fd_check(lambda a: loss(**{name: a}), kw[name], g[name], rng, label=name)
