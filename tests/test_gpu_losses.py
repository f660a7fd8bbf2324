"""GPU tests of the photometric training loss (pf3plat_b200/losses.py -> csrc/gs_losses.cu) against the fp64 oracle
(oracle/ssim_loss_oracle.py) and the reference's own loss code (tests/golden/ssim_loss.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import ssim_loss_oracle as so
from pf3plat_b200 import losses
from pf3plat_b200.synthetic import make_scene, make_target
from tests.util import check_grad

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssim_loss.npz")
VALUE_TOL = 1e-5


def _render(n, h, w, seed):
    """n synthetic-scene renders on a black background: sparse splats leave large flat regions where u = v = 0."""
    from pf3plat_b200.render import render_views
    d = make_scene(60 + (h * w) // 400, n, h, w, seed=seed).to(DEV)
    with torch.no_grad():
        return render_views(d.extrinsics, d.intrinsics, d.near, d.far, d.image_shape, d.background, d.means[None],
                            d.covariances[None], d.harmonics[None], d.opacities[None]).float()


def _pair(kind, n, c, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "noise":
        return torch.rand(n, c, h, w, generator=g), torch.rand(n, c, h, w, generator=g)
    if kind == "out_of_range":
        return -0.1 + 1.3 * torch.rand(n, c, h, w, generator=g), -0.1 + 1.3 * torch.rand(n, c, h, w, generator=g)
    if kind == "render":
        assert c == 3
        y = _render(n, h, w, seed).cpu()
        x = _render(n, h, w, seed + 1).cpu()   # another cloud seen from the same cameras
        return x, y
    raise KeyError(kind)


def _gpu_per_image(x, y, ws, wm):
    xg = x.to(DEV).requires_grad_(True)
    yg = y.to(DEV).requires_grad_(True)
    s, m = losses._per_image(xg, yg)
    ((s * ws.to(DEV)).sum() + (m * wm.to(DEV)).sum()).backward()
    return s.detach().cpu(), m.detach().cpu(), xg.grad.cpu(), yg.grad.cpu()


def _check_against_oracle(x, y, label, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = x.shape[0]
    ws, wm = torch.randn(n, generator=g), torch.randn(n, generator=g)
    s, m, gx, gy = _gpu_per_image(x, y, ws, wm)
    so_, mo, gxo, gyo = so.per_image_with_grads(x, y, d_ssim=ws, d_mse=wm)
    es, em = float((s.double() - so_).abs().max()), float((m.double() - mo).abs().max())
    print(f"[ssim-loss] {label}: worst |ssim - oracle| {es:.2e}, |mse - oracle| {em:.2e}")
    assert es <= VALUE_TOL and em <= VALUE_TOL
    check_grad(f"{label} dL/dpred", gx.reshape(-1), gxo.reshape(-1).numpy())
    check_grad(f"{label} dL/dgt", gy.reshape(-1), gyo.reshape(-1).numpy())


SHAPES = [  # (kind, n, c, h, w)
    ("noise", 1, 1, 1, 1), ("noise", 3, 3, 1, 40), ("out_of_range", 2, 4, 40, 1), ("noise", 2, 3, 5, 7),
    ("noise", 4, 4, 10, 10), ("noise", 2, 1, 11, 11), ("render", 2, 3, 12, 300), ("out_of_range", 2, 3, 33, 250),
    ("noise", 60, 3, 16, 20), ("render", 3, 3, 256, 256), ("noise", 1, 3, 512, 512), ("render", 1, 3, 512, 512),
    ("out_of_range", 2, 1, 256, 256), ("render", 14, 3, 64, 64),
]


@pytest.mark.parametrize("kind,n,c,h,w", SHAPES)
def test_values_and_gradients_match_the_fp64_oracle(kind, n, c, h, w):
    x, y = _pair(kind, n, c, h, w, seed=h * 1000 + w)
    _check_against_oracle(x, y, f"{kind} {n}x{c}x{h}x{w}")


@pytest.mark.parametrize("name", ["random", "render", "out_of_range", "tiny_5x7", "tiny_1x1", "batch_37x45"])
def test_the_reference_fixture(name):
    z = np.load(GOLDEN)
    x, y, w = (torch.from_numpy(z[f"{name}/{k}"]) for k in ("x", "y", "w_img"))
    s, m, gx, gy = _gpu_per_image(x, y, w.float(), torch.zeros(x.shape[0]))
    es = float(np.abs(s.numpy() - z[f"{name}/f64/ssim_img"]).max())
    em = abs(float(m.double().mean()) - float(z[f"{name}/f64/loss_mse"]))
    print(f"[ssim-loss] fixture {name}: worst |ssim - reference fp64| {es:.2e}, |mse - reference| {em:.2e}")
    assert es <= VALUE_TOL and em <= VALUE_TOL
    check_grad(f"fixture {name} dL/dpred", gx.reshape(-1), z[f"{name}/f64/grad_x"].reshape(-1))
    check_grad(f"fixture {name} dL/dgt", gy.reshape(-1), z[f"{name}/f64/grad_y"].reshape(-1))


@pytest.mark.parametrize("n,c,h,w", [(2, 3, 16, 16), (1, 1, 1, 1), (2, 3, 5, 7), (2, 3, 256, 256)])
def test_identical_pairs_give_one_and_a_vanishing_gradient(n, c, h, w):
    """The exact gradient is 0; in float32 it is rounding noise, held far below the gradient of a differing pair."""
    x = torch.rand(n, c, h, w, generator=torch.Generator().manual_seed(7))
    z = torch.zeros(n)
    s, m, gx, gy = _gpu_per_image(x, x.clone(), torch.ones(n), z)
    _, _, gx_ref, _ = _gpu_per_image(x, torch.rand(n, c, h, w, generator=torch.Generator().manual_seed(8)), torch.ones(n), z)
    worst = float(max(gx.abs().max(), gy.abs().max()))
    print(f"[ssim-loss] identical {n}x{c}x{h}x{w}: |1 - ssim| {float((s - 1).abs().max()):.2e}, max |grad| {worst:.2e} "
          f"vs {float(gx_ref.abs().max()):.2e} for a differing pair")
    assert float((s - 1).abs().max()) <= 1e-6 and float(m.abs().max()) == 0.0
    assert worst <= 1e-3 * float(gx_ref.abs().max())
    z = np.load(GOLDEN)    # the reference's own identical pair
    s, _, _, _ = _gpu_per_image(torch.from_numpy(z["identical/x"]), torch.from_numpy(z["identical/y"]), torch.ones(2),
                                torch.zeros(2))
    assert float((s - 1).abs().max()) <= 1e-6


def test_photometric_loss_equals_separate_ssim_and_mse():
    x, y = _pair("render", 4, 3, 64, 96, seed=3)
    a = x.to(DEV).requires_grad_(True)
    b = y.to(DEV).requires_grad_(True)
    mse_term, ssim_term = losses.photometric_loss(a, b)
    (mse_term + ssim_term).backward()
    a2 = x.to(DEV).requires_grad_(True)
    b2 = y.to(DEV).requires_grad_(True)
    s = losses.ssim(a2, b2)
    m = ((a2 - b2) ** 2).mean()
    (1.0 * m + 0.1 * (1 - s)).backward()
    assert torch.equal(ssim_term, 0.1 * (1 - s.detach()))
    assert abs(float(mse_term.detach()) - float(m.detach())) <= 1e-6 * float(m.detach())
    for ours, sep in ((a.grad, a2.grad), (b.grad, b2.grad)):
        check_grad("photometric_loss vs ssim + mse", ours.reshape(-1), sep.reshape(-1).cpu().numpy())
    # the weights scale the terms and their gradients
    m5, s5 = losses.photometric_loss(a.detach(), b.detach(), mse_weight=5.0, ssim_weight=2.0)
    assert torch.allclose(m5, 5 * mse_term.detach()) and torch.allclose(s5, 20 * ssim_term.detach())


@pytest.mark.parametrize("term", ["mse", "ssim"])
def test_backward_through_one_term_only(term):
    x, y = _pair("noise", 3, 3, 40, 50, seed=9)
    a = x.to(DEV).requires_grad_(True)
    b = y.to(DEV).requires_grad_(True)
    mse_term, ssim_term = losses.photometric_loss(a, b)
    (mse_term if term == "mse" else ssim_term).backward()
    n = x.shape[0]
    ds = torch.zeros(n) if term == "mse" else torch.full((n,), -0.1 / n)
    dm = torch.full((n,), 1.0 / n) if term == "mse" else None
    _, _, gxo, gyo = so.per_image_with_grads(x, y, d_ssim=ds, d_mse=dm)
    check_grad(f"{term} only dL/dpred", a.grad.reshape(-1).cpu(), gxo.reshape(-1).numpy())
    check_grad(f"{term} only dL/dgt", b.grad.reshape(-1).cpu(), gyo.reshape(-1).numpy())


def test_only_the_requested_input_gradient_is_computed():
    x, y = _pair("noise", 2, 3, 33, 47, seed=10)
    a = x.to(DEV).requires_grad_(True)
    b = y.to(DEV)
    sum(losses.photometric_loss(a, b)).backward()
    a2 = x.to(DEV).requires_grad_(True)
    b2 = y.to(DEV).requires_grad_(True)
    sum(losses.photometric_loss(a2, b2)).backward()
    assert torch.equal(a.grad, a2.grad)


@pytest.mark.parametrize("b,v", [(1, 5), (2, 3), (3, 5)])
def test_strided_inner_views_equal_their_contiguous_copy_bitwise(b, v):
    g = torch.Generator().manual_seed(11)
    color = torch.rand(b, v, 3, 64, 80, generator=g).to(DEV).requires_grad_(True)
    target = torch.rand(b, v, 3, 64, 80, generator=g).to(DEV)
    m1, s1 = losses.photometric_loss(color[:, 1:-1], target[:, 1:-1])
    (m1 + s1).backward()
    inner = color.detach()[:, 1:-1].contiguous().requires_grad_(True)
    m2, s2 = losses.photometric_loss(inner, target[:, 1:-1].contiguous())
    (m2 + s2).backward()
    assert torch.equal(m1, m2) and torch.equal(s1, s2)
    assert torch.equal(color.grad[:, 1:-1], inner.grad)
    assert float(color.grad[:, 0].abs().max()) == 0.0 and float(color.grad[:, -1].abs().max()) == 0.0
    per = losses.ssim(color.detach()[:, 1:-1], target[:, 1:-1], size_average=False)
    assert per.shape == (b, v - 2)


def test_two_runs_are_bit_identical():
    x, y = _pair("render", 3, 3, 256, 256, seed=12)
    outs = []
    for _ in range(2):
        a = x.to(DEV).requires_grad_(True)
        b = y.to(DEV).requires_grad_(True)
        m, s = losses.photometric_loss(a, b)
        (m + s).backward()
        outs.append((m.detach(), s.detach(), a.grad, b.grad))
    for p, q in zip(*outs):
        assert torch.equal(p, q)


def test_inputs_must_be_float32():
    x = torch.rand(1, 3, 8, 8, device=DEV, dtype=torch.float64)
    with pytest.raises(TypeError, match="float32"):
        losses.ssim(x, x)


def test_decoder_to_loss_chain_matches_the_oracle_loss_gradient():
    """decoder_forward -> photometric_loss on color[:, 1:-1] -> backward to the Gaussians, against the same rasterizer
    backward fed with dL/dcolor from the fp64 oracle."""
    from pf3plat_b200.render import decoder_forward
    b, v, hw, P = 2, 3, (96, 128), 3000
    scs = [make_scene(P, v, *hw, seed=40 + k).to(DEV) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs])
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), 1.0, device=DEV), torch.full((b, v), 100.0, device=DEV)
    bg = torch.zeros(3, device=DEV)
    base = [st(n) for n in ("means", "covariances", "harmonics", "opacities")]
    target = make_target(b * v, *hw, seed=5).to(DEV).reshape(b, v, 3, *hw)

    leaves = [t.clone().requires_grad_(True) for t in base]
    color, _ = decoder_forward(*leaves, ext, intr, nr, fr, hw, bg)
    color.retain_grad()
    mse_term, ssim_term = losses.photometric_loss(color[:, 1:-1], target[:, 1:-1])
    (mse_term + ssim_term).backward()

    # dL/dcolor of the same loss from the fp64 oracle, on the rendered colours
    x = color.detach()[:, 1:-1].reshape(-1, 3, *hw).cpu()
    y = target[:, 1:-1].reshape(-1, 3, *hw).cpu()
    n = x.shape[0]
    _, _, dx, _ = so.per_image_with_grads(x, y, d_ssim=torch.full((n,), -0.1 / n), d_mse=torch.full((n,), 1.0 / n))
    dcolor = torch.zeros_like(color)
    dcolor[:, 1:-1] = dx.reshape(b, v - 2, 3, *hw).float().to(DEV)
    check_grad("chain dL/dcolor", color.grad.reshape(-1).cpu(), dcolor.reshape(-1).cpu().numpy())
    leaves_o = [t.clone().requires_grad_(True) for t in base]
    color_o, _ = decoder_forward(*leaves_o, ext, intr, nr, fr, hw, bg)
    color_o.backward(dcolor)
    for name, ours, ref in zip(("means", "covariances", "harmonics", "opacities"), leaves, leaves_o):
        check_grad(f"chain dL/d{name}", ours.grad.reshape(b * P, -1).cpu(), ref.grad.reshape(b * P, -1).cpu().numpy())
