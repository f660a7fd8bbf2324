"""GPU tests of LPIPS-VGG's BF16 path (LPIPS(precision="bf16") -> k_conv3x3_wgmma and the BF16 instantiations in
csrc/gs_lpips.cu) against the fp64 oracle (oracle/lpips_oracle.py).

The bound is relative to what PyTorch gets for the same module under torch.autocast(dtype=torch.bfloat16) (cuDNN BF16
convolutions with fp32 accumulation, the mixed precision a user of the `lpips` package gets):
  value:    |ours - fp64| <= max(2 max|torch_bf16 - fp64|, 1e-3 |fp64| + 1e-5)      per image
  gradient: ||ours - fp64|| / ||fp64|| <= max(2 (the same for torch_bf16), 1e-2)
"""
import pytest
import torch

from oracle import lpips_oracle as lo
from pf3plat_b200 import lpips as pl
from pf3plat_b200.synthetic import make_scene, make_target
from tests import test_gpu_lpips as tl

pytestmark = pytest.mark.gpu
DEV = tl.DEV
SD = tl.SD
_pair, _rel = tl._pair, tl._rel


@pytest.fixture(scope="module")
def model():
    return pl.LPIPS(net="vgg", weights=SD, precision="bf16").to(DEV)


@pytest.fixture
def restore_precision():
    prev = pl.get_precision()
    yield
    pl.set_precision(prev)


def _torch_bf16(x0, x1, normalize, dout, sd=SD):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        return lo.with_grads(x0, x1, sd, normalize, dout, device=DEV, dtype=torch.float32)


def _ours(model, x0, x1, normalize, dout, which):
    a = x0.clone().requires_grad_(which == 0)
    b = x1.clone().requires_grad_(which == 1)
    v = model(a, b, normalize=normalize)
    assert v.shape == (x0.shape[0], 1, 1, 1) and v.dtype == torch.float32
    (v.reshape(-1) * dout.to(DEV)).sum().backward()
    g = (a if which == 0 else b).grad
    assert g.dtype == torch.float32
    return v.detach().reshape(-1).cpu().double(), g.cpu().double()


@pytest.mark.parametrize("kind,n,h,w,normalize,which", tl.CASES)
def test_values_and_gradients_against_the_fp64_oracle(model, kind, n, h, w, normalize, which):
    x0, x1 = _pair(kind, n, h, w, seed=h * 1000 + w + n)
    dout = 0.5 + torch.rand(n, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    v, g = _ours(model, x0, x1, normalize, dout, which)
    v64, *g64 = lo.with_grads(x0, x1, SD, normalize, dout, device=DEV, dtype=torch.float64)
    vb, *gb = _torch_bf16(x0, x1, normalize, dout)
    g64, gb = g64[which], gb[which].double()
    err = (v - v64).abs()
    err_b = float((vb.double() - v64).abs().max())
    bound = torch.maximum(torch.full_like(v64, 2 * err_b), 1e-3 * v64.abs() + 1e-5)
    rel, rel_b = _rel(g, g64), _rel(gb, g64)
    print(f"[lpips-bf16] {kind} {n}x3x{h}x{w} normalize={normalize} d/din{which}: value fp64 {v64.numpy()[:3]} | "
          f"|ours-fp64| max {float(err.max()):.2e} (torch_bf16 {err_b:.2e}) | grad rel-L2 ours {rel:.2e} "
          f"torch_bf16 {rel_b:.2e}")
    assert bool((err <= bound).all()), (err, bound)
    assert rel <= max(2 * rel_b, 1e-2), (rel, rel_b)


@pytest.mark.parametrize("n,h,w", [(2, 37, 53), (14, 256, 256)])
def test_identical_pairs_give_exactly_zero(model, n, h, w):
    x = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(5)).to(DEV)
    a = x.clone().requires_grad_(True)
    b = x.clone().requires_grad_(True)
    v = model(a, b, normalize=True)
    v.sum().backward()
    assert float(v.detach().abs().max()) == 0.0
    assert float(a.grad.abs().max()) == 0.0 and float(b.grad.abs().max()) == 0.0


def test_two_runs_are_bit_identical(model):
    x0, x1 = _pair("render", 4, 64, 96, seed=3)
    outs = []
    for _ in range(2):
        a, b = x0.clone().requires_grad_(True), x1.clone().requires_grad_(True)
        v = model(a, b, normalize=True)
        v.sum().backward()
        outs.append((v.detach(), a.grad, b.grad))
    for p, q in zip(*outs):
        assert torch.equal(p, q)


@pytest.mark.parametrize("b,v", [(1, 5), (4, 3)])
def test_a_strided_view_gives_the_bits_of_its_contiguous_copy(model, b, v):
    g = torch.Generator().manual_seed(b * 10 + v)
    color = torch.rand(b, v, 3, 48, 64, generator=g).to(DEV).requires_grad_(True)
    target = torch.rand(b, v, 3, 48, 64, generator=g).to(DEV)
    out = model(color[:, 1:-1], target[:, 1:-1], normalize=True)
    out.sum().backward()
    inner = color.detach()[:, 1:-1].contiguous().reshape(-1, 3, 48, 64).requires_grad_(True)
    out2 = model(inner, target[:, 1:-1].reshape(-1, 3, 48, 64), normalize=True)
    out2.sum().backward()
    assert torch.equal(out.reshape(-1), out2.reshape(-1))
    assert torch.equal(color.grad[:, 1:-1].reshape(-1, 3, 48, 64), inner.grad)
    assert float(color.grad[:, 0].abs().max()) == 0.0 and float(color.grad[:, -1].abs().max()) == 0.0


def test_only_the_requested_gradients_are_computed_and_they_do_not_depend_on_the_other(model):
    x0, x1 = _pair("noise", 3, 40, 36, seed=4)
    grads = {}
    for need in ((True, False), (False, True), (True, True)):
        a, b = x0.clone().requires_grad_(need[0]), x1.clone().requires_grad_(need[1])
        model(a, b).sum().backward()
        assert (a.grad is not None) == need[0] and (b.grad is not None) == need[1]
        grads[need] = (a.grad, b.grad)
    assert torch.equal(grads[(True, False)][0], grads[(True, True)][0])
    assert torch.equal(grads[(False, True)][1], grads[(True, True)][1])
    with torch.no_grad():
        v = model(x0, x1)
    assert torch.equal(v, model(x0, x1).detach())


def test_a_tap_with_zero_norm_gives_a_finite_gradient():
    sd = dict(SD)
    sd["net.slice5.28.bias"] = torch.full((512,), -1e3)
    m = pl.LPIPS(weights=sd, precision="bf16").to(DEV)
    x0, x1 = _pair("noise", 2, 48, 40, seed=6)
    a = x0.clone().requires_grad_(True)
    v = m(a, x1)
    v.sum().backward()
    v64, g64, _ = lo.with_grads(x0, x1, sd, False, device=DEV)
    _, gb, _ = _torch_bf16(x0, x1, False, None, sd)
    rel, rel_b = _rel(a.grad.cpu().double(), g64), _rel(gb.double(), g64)
    print(f"[lpips-bf16] s = 0 at relu5_3: value {v.detach().reshape(-1).cpu().numpy()} vs fp64 {v64.numpy()}; "
          f"grad rel-L2 ours {rel:.2e}, torch_bf16 {rel_b:.2e}")
    assert bool(torch.isfinite(v).all()) and bool(torch.isfinite(a.grad).all())
    assert rel <= max(2 * rel_b, 1e-2)


def test_a_nan_pixel_makes_only_its_image_nan(model):
    x0, x1 = _pair("noise", 3, 40, 48, seed=7)
    base = model(x0, x1).detach().reshape(-1)
    bad = x0.clone()
    bad[1, 2, 17, 30] = float("nan")
    a = bad.clone().requires_grad_(True)
    v = model(a, x1).reshape(-1)
    v.sum().backward()
    assert bool(torch.isnan(v[1])) and bool(torch.isfinite(base).all())
    assert torch.equal(v.detach()[[0, 2]], base[[0, 2]])
    assert bool(torch.isfinite(a.grad[[0, 2]]).all())


def test_weight_changes_repack_the_bf16_weights_exactly_when_the_weights_change():
    x0, x1 = _pair("noise", 2, 32, 32, seed=8)
    m = pl.LPIPS(weights=SD, precision="bf16").to(DEV)
    base = tl._module_value(m, x0, x1)
    pack = m._packs[(DEV, "bf16")][1]
    assert torch.equal(base, tl._module_value(m, x0, x1))
    assert m._packs[(DEV, "bf16")][1] is pack  # no change, no repack
    with torch.no_grad():
        m.net.slice3._modules["12"].weight.mul_(3.0)  # conv3_2: a BF16-packed convolution
    changed = tl._module_value(m, x0, x1)
    assert m._packs[(DEV, "bf16")][1] is not pack
    assert not torch.equal(changed, base)
    ref = pl.LPIPS(weights=pl.canonical_state_dict(m.state_dict()), precision="bf16").to(DEV)
    assert torch.equal(changed, tl._module_value(ref, x0, x1))
    with torch.no_grad():
        m.net.slice3._modules["12"].weight.div_(3.0)
    assert torch.allclose(tl._module_value(m, x0, x1), base, rtol=1e-3)


def test_the_default_path_is_untouched(restore_precision):
    x0, x1 = _pair("render", 2, 64, 80, seed=9)
    pl.set_precision("tf32")
    plain, tf32 = pl.LPIPS(weights=SD).to(DEV), pl.LPIPS(weights=SD, precision="tf32").to(DEV)
    a, b = x0.clone().requires_grad_(True), x0.clone().requires_grad_(True)
    va, vb = plain(a, x1), tf32(b, x1)
    va.sum().backward()
    vb.sum().backward()
    assert torch.equal(va, vb) and torch.equal(a.grad, b.grad)
    # the setter switches modules that never mention precision, and only those
    pl.set_precision("bf16")
    assert not torch.equal(plain(x0, x1), va) and torch.equal(tf32(x0, x1), vb.detach())
    assert torch.equal(plain(x0, x1), pl.LPIPS(weights=SD, precision="bf16").to(DEV)(x0, x1))


def test_compute_lpips_does_not_follow_the_setter(monkeypatch, restore_precision):
    from pf3plat_b200 import metrics
    monkeypatch.setattr(pl, "_package_state_dict", lambda: SD)
    metrics.get_lpips.cache_clear()
    gt, pr = _pair("render", 3, 64, 80, seed=9)
    pl.set_precision("tf32")
    off = metrics.compute_lpips(gt, pr)
    pl.set_precision("bf16")
    on = metrics.compute_lpips(gt, pr)
    metrics.get_lpips.cache_clear()
    assert torch.equal(off, on)


def test_render_to_loss_chain_matches_the_oracle_image_gradient():
    """decoder_forward -> photometric_loss + 0.1 LPIPS-BF16 on color[:, 1:-1] -> backward to the Gaussians, against the
    same chain fed dL/dcolor from the fp64 oracle (and, for the bound, from PyTorch under BF16 autocast)."""
    from oracle import ssim_loss_oracle as so
    from pf3plat_b200 import losses
    from pf3plat_b200.render import decoder_forward
    b, v, hw, P = 2, 3, (64, 96), 3000
    scs = [make_scene(P, v, *hw, seed=50 + k).to(DEV) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs])
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), 1.0, device=DEV), torch.full((b, v), 100.0, device=DEV)
    bg = torch.zeros(3, device=DEV)
    base = [st(n) for n in ("means", "covariances", "harmonics", "opacities")]
    target = make_target(b * v, *hw, seed=6).to(DEV).reshape(b, v, 3, *hw)
    model = pl.LPIPS(weights=SD, precision="bf16").to(DEV)

    leaves = [t.clone().requires_grad_(True) for t in base]
    color, _ = decoder_forward(*leaves, ext, intr, nr, fr, hw, bg)
    color.retain_grad()
    mse_term, ssim_term = losses.photometric_loss(color[:, 1:-1], target[:, 1:-1])
    lp = model(color[:, 1:-1].reshape(-1, 3, *hw), target[:, 1:-1].reshape(-1, 3, *hw), normalize=True)
    (mse_term + ssim_term + 0.1 * lp.mean()).backward()

    x = color.detach()[:, 1:-1].reshape(-1, 3, *hw)
    y = target[:, 1:-1].reshape(-1, 3, *hw)
    n = x.shape[0]
    _, _, dphoto, _ = so.per_image_with_grads(x.cpu(), y.cpu(), d_ssim=torch.full((n,), -0.1 / n), d_mse=torch.full((n,), 1.0 / n))
    dout = torch.full((n,), 0.1 / n, dtype=torch.float64)
    grads = {}
    for tag in ("fp64", "torch_bf16"):
        if tag == "fp64":
            _, dl, _ = lo.with_grads(x, y, SD, True, dout, device=DEV, dtype=torch.float64)
        else:
            _, dl, _ = _torch_bf16(x, y, True, dout)
        dcolor = torch.zeros_like(color)
        dcolor[:, 1:-1] = (dphoto + dl.double()).reshape(b, v - 2, 3, *hw).float().to(DEV)
        leaves_o = [t.clone().requires_grad_(True) for t in base]
        color_o, _ = decoder_forward(*leaves_o, ext, intr, nr, fr, hw, bg)
        color_o.backward(dcolor)
        grads[tag] = (dcolor, [t.grad for t in leaves_o])
    ref_c, ref_l = grads["fp64"]
    bf_c, bf_l = grads["torch_bf16"]
    rc, rc_b = _rel(color.grad.double(), ref_c.double()), _rel(bf_c.double(), ref_c.double())
    print(f"[lpips-bf16] chain dL/dcolor rel-L2 ours {rc:.2e}, torch_bf16 {rc_b:.2e}")
    assert rc <= max(2 * rc_b, 1e-2)
    for name, ours, ref, bf in zip(("means", "covariances", "harmonics", "opacities"), leaves, ref_l, bf_l):
        r, r_b = _rel(ours.grad.double(), ref.double()), _rel(bf.double(), ref.double())
        print(f"[lpips-bf16] chain dL/d{name} rel-L2 ours {r:.2e}, torch_bf16 {r_b:.2e}")
        assert r <= max(2 * r_b, 1e-2), name
