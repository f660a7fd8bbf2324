"""GPU tests of LPIPS-VGG (pf3plat_b200/lpips.py -> csrc/gs_lpips.cu) against the fp64 oracle (oracle/lpips_oracle.py).

Element-wise 1e-3 is not a meaningful bound after 13 TF32 convolutions, so the bound is relative to what PyTorch gets
today for the same module (cuDNN with TF32 allowed, its default on an H100):
  value:    |ours - fp64| <= max(2 max|torch_tf32 - fp64|, 1e-4 |fp64| + 1e-6)      per image
  gradient: ||ours - fp64|| / ||fp64|| <= max(2 (the same for torch_tf32), 1e-3)
"""
import os

import numpy as np
import pytest
import torch

from oracle import lpips_oracle as lo
from pf3plat_b200 import lpips as pl
from pf3plat_b200.synthetic import make_scene, make_target

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lpips_small.npz")
SD = lo.random_state_dict(11)


@pytest.fixture(scope="module")
def model():
    return pl.LPIPS(net="vgg", weights=SD).to(DEV)


def _render(n, h, w, seed):
    from pf3plat_b200.render import render_views
    d = make_scene(60 + (h * w) // 400, n, h, w, seed=seed).to(DEV)
    with torch.no_grad():
        return render_views(d.extrinsics, d.intrinsics, d.near, d.far, d.image_shape, d.background, d.means[None],
                            d.covariances[None], d.harmonics[None], d.opacities[None]).float()


def _pair(kind, n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "noise":
        return torch.rand(n, 3, h, w, generator=g).to(DEV), torch.rand(n, 3, h, w, generator=g).to(DEV)
    if kind == "out_of_range":
        return ((-0.1 + 1.3 * torch.rand(n, 3, h, w, generator=g)).to(DEV),
                (-0.1 + 1.3 * torch.rand(n, 3, h, w, generator=g)).to(DEV))
    if kind == "render":
        return _render(n, h, w, seed), _render(n, h, w, seed + 1)
    raise KeyError(kind)


def _torch(x0, x1, normalize, dout, dtype, tf32, sd=SD):
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        return lo.with_grads(x0, x1, sd, normalize, dout, device=DEV, dtype=dtype)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _ours(model, x0, x1, normalize, dout, which):
    a = x0.clone().requires_grad_(which == 0)
    b = x1.clone().requires_grad_(which == 1)
    v = model(a, b, normalize=normalize)
    assert v.shape == (x0.shape[0], 1, 1, 1)
    (v.reshape(-1) * dout.to(DEV)).sum().backward()
    return v.detach().reshape(-1).cpu().double(), (a if which == 0 else b).grad.cpu().double()


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def check_against_oracle(model, x0, x1, normalize, which, label, seed=0):
    n = x0.shape[0]
    dout = 0.5 + torch.rand(n, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    v, g = _ours(model, x0, x1, normalize, dout, which)
    v64, *g64 = _torch(x0, x1, normalize, dout, torch.float64, False)
    vt, *gt = _torch(x0, x1, normalize, dout, torch.float32, True)
    vf, *gf = _torch(x0, x1, normalize, dout, torch.float32, False)
    g64, gt, gf = g64[which], gt[which].double(), gf[which].double()
    err = (v - v64).abs()
    err_t = float((vt.double() - v64).abs().max())
    bound = torch.maximum(torch.full_like(v64, 2 * err_t), 1e-4 * v64.abs() + 1e-6)
    rel, rel_t = _rel(g, g64), _rel(gt, g64)
    print(f"[lpips] {label}: value fp64 {v64.numpy()[:3]} | |ours-fp64| max {float(err.max()):.2e} "
          f"(torch_tf32 {err_t:.2e}, torch_fp32 {float((vf.double() - v64).abs().max()):.2e}, "
          f"ours vs torch_fp32 {float((v - vf.double()).abs().max()):.2e}) | grad rel-L2 ours {rel:.2e} "
          f"torch_tf32 {rel_t:.2e} torch_fp32 {_rel(gf, g64):.2e} ours vs torch_fp32 {_rel(g, gf):.2e}")
    assert bool((err <= bound).all()), (err, bound)
    assert rel <= max(2 * rel_t, 1e-3), (rel, rel_t)


CASES = [  # (kind, n, h, w, normalize, gradient of in0 (0) or in1 (1))
    ("noise", 1, 16, 16, True, 0),
    ("out_of_range", 2, 37, 53, False, 1),
    ("render", 3, 17, 130, True, 1),
    ("render", 4, 64, 64, False, 0),
    ("noise", 14, 256, 256, True, 0),
    ("render", 1, 512, 512, True, 1),
    ("out_of_range", 2, 256, 256, True, 0),
    ("noise", 3, 17, 130, False, 0),
]


@pytest.mark.parametrize("kind,n,h,w,normalize,which", CASES)
def test_values_and_gradients_against_the_fp64_oracle(model, kind, n, h, w, normalize, which):
    x0, x1 = _pair(kind, n, h, w, seed=h * 1000 + w + n)
    check_against_oracle(model, x0, x1, normalize, which, f"{kind} {n}x3x{h}x{w} normalize={normalize} d/din{which}")


@pytest.mark.parametrize("n,h,w", [(2, 37, 53), (14, 256, 256)])
def test_identical_pairs_give_exactly_zero(model, n, h, w):
    x = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(5)).to(DEV)
    a = x.clone().requires_grad_(True)
    b = x.clone().requires_grad_(True)
    v = model(a, b, normalize=True)
    v.sum().backward()
    print(f"[lpips] identical {n}x3x{h}x{w}: max |value| {float(v.abs().max()):.1e}, max |grad| "
          f"{float(max(a.grad.abs().max(), b.grad.abs().max())):.1e}")
    assert float(v.abs().max()) == 0.0
    assert float(a.grad.abs().max()) == 0.0 and float(b.grad.abs().max()) == 0.0


def test_the_golden_fixture():
    """The recorded fp64 values and gradients, under the bound of the module docstring (PyTorch's TF32 run of the same
    weights gives the scale)."""
    z = np.load(GOLDEN)
    sd = lo.random_state_dict(int(z["weight_seed"]))
    m = pl.LPIPS(weights=sd).to(DEV)
    for name in ("noise_16x16", "ragged_17x23", "out_of_range_33x19", "noise_40x48"):
        x0, x1 = (torch.from_numpy(z[f"{name}/{k}"]).to(DEV) for k in ("x0", "x1"))
        dout = torch.from_numpy(z[f"{name}/dout"])
        a, b = x0.clone().requires_grad_(True), x1.clone().requires_grad_(True)
        v = m(a, b, normalize=bool(z[f"{name}/normalize"])).reshape(-1)
        (v * dout.float().to(DEV)).sum().backward()
        v64, g064, g164 = (torch.from_numpy(z[f"{name}/{k}"]) for k in ("value", "grad0", "grad1"))
        vt, gt0, gt1 = _torch(x0, x1, bool(z[f"{name}/normalize"]), dout, torch.float32, True, sd)
        err = (v.detach().cpu().double() - v64).abs()
        err_t = float((vt.double() - v64).abs().max())
        r0, r1 = _rel(a.grad.cpu().double(), g064), _rel(b.grad.cpu().double(), g164)
        t0, t1 = _rel(gt0.double(), g064), _rel(gt1.double(), g164)
        print(f"[lpips] fixture {name}: |value - fp64| {float(err.max()):.2e} (torch_tf32 {err_t:.2e}), grad rel-L2 "
              f"{r0:.2e} / {r1:.2e} (torch_tf32 {t0:.2e} / {t1:.2e})")
        assert bool((err <= torch.clamp(1e-4 * v64.abs() + 1e-6, min=2 * err_t)).all())
        assert r0 <= max(2 * t0, 1e-3) and r1 <= max(2 * t1, 1e-3)


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
    assert out.shape == (b, v - 2, 1, 1, 1)
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
    with torch.no_grad():   # forward only: no saved activations
        v = model(x0, x1)
    assert torch.equal(v, model(x0, x1).detach())


def test_a_tap_with_zero_norm_gives_a_finite_gradient():
    """conv5_3's bias kills relu5_3 everywhere, so every pixel of the last tap has s = 0 while the other four taps still
    differ.  There autograd's dL/df is NaN (sqrt's backward at 0) and ReLU's backward selects 0 over it; ours defines
    dL/df = g / 1e-10 (DESIGN.md 5.10), which the same mask removes.  Both input gradients are finite and agree."""
    sd = dict(SD)
    sd["net.slice5.28.bias"] = torch.full((512,), -1e3)
    m = pl.LPIPS(weights=sd).to(DEV)
    x0, x1 = _pair("noise", 2, 48, 40, seed=6)
    a = x0.clone().requires_grad_(True)
    v = m(a, x1)
    v.sum().backward()
    v64, g64, _ = lo.with_grads(x0, x1, sd, False, device=DEV)
    _, gt, _ = _torch(x0, x1, False, None, torch.float32, True, sd)
    rel, rel_t = _rel(a.grad.cpu().double(), g64), _rel(gt.double(), g64)
    print(f"[lpips] s = 0 at relu5_3: value {v.detach().reshape(-1).cpu().numpy()} vs fp64 {v64.numpy()}; grad rel-L2 "
          f"ours {rel:.2e}, torch_tf32 {rel_t:.2e}")
    assert float(v64.abs().min()) > 0
    assert torch.allclose(v.detach().reshape(-1).cpu().double(), v64, rtol=1e-3, atol=1e-7)
    assert bool(torch.isfinite(a.grad).all()) and bool(torch.isfinite(g64).all())
    assert rel <= max(2 * rel_t, 1e-3)


def _module_value(m, x0, x1):
    return m(x0, x1, normalize=True).detach().reshape(-1)


def test_weight_changes_repack_exactly_when_the_weights_change():
    x0, x1 = _pair("noise", 2, 32, 32, seed=8)
    m = pl.LPIPS(weights=SD).to(DEV)
    base = _module_value(m, x0, x1)
    assert torch.equal(base, _module_value(m, x0, x1))
    # convert_to_buffer as PF3plat does it: every parameter re-registered as a (non-persistent) buffer
    def to_buffers(module):
        for child in list(module.children()):
            to_buffers(child)
        for name, t in (*module.named_parameters(recurse=False), *module.named_buffers(recurse=False)):
            value = t.detach().clone()
            delattr(module, name)
            module.register_buffer(name, value, persistent=False)
    to_buffers(m)
    assert not list(m.parameters())
    assert torch.equal(base, _module_value(m, x0, x1))
    # an in-place change of one weight
    with torch.no_grad():
        m.lin2.model["1"].weight.mul_(3.0)
    changed = _module_value(m, x0, x1)
    assert not torch.equal(changed, base)
    with torch.no_grad():
        m.lin2.model["1"].weight.div_(3.0)
    assert torch.allclose(_module_value(m, x0, x1), base, rtol=1e-6)
    # load_state_dict with other weights, then back
    m2 = pl.LPIPS(weights=SD).to(DEV)
    other = lo.random_state_dict(12)
    m2.load_state_dict(pl.canonical_state_dict(other))
    v_other = _module_value(m2, x0, x1)
    ref_other = pl.LPIPS(weights=other).to(DEV)
    assert torch.equal(v_other, _module_value(ref_other, x0, x1)) and not torch.equal(v_other, base)
    m2.load_state_dict(pl.canonical_state_dict(SD))
    assert torch.equal(_module_value(m2, x0, x1), base)
    # .to(): a module moved to the CPU and back packs again from the new tensors
    m2.to("cpu")
    m2.to(DEV)
    assert torch.equal(_module_value(m2, x0, x1), base)
    # a replaced tensor
    m2.net.slice1._modules["0"].bias = torch.nn.Parameter(torch.zeros(64, device=DEV))
    assert not torch.equal(_module_value(m2, x0, x1), base)


def test_bad_inputs_are_refused(model):
    x = torch.rand(2, 3, 32, 32, device=DEV)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model(x.cpu(), x.cpu())
    with pytest.raises(TypeError, match="float32"):
        model(x.double(), x.double())
    with pytest.raises(ValueError):
        model(x, x[:1])
    with pytest.raises(ValueError):
        model(x[:, :, :15], x[:, :, :15])
    with pytest.raises(ValueError):
        model(x[:, :, :, :8], x[:, :, :, :8])
    with pytest.raises(ValueError):
        model(x[:, :1], x[:, :1])


def test_compute_lpips_has_the_reference_signature(monkeypatch):
    from pf3plat_b200 import metrics
    monkeypatch.setattr(pl, "_package_state_dict", lambda: SD)
    metrics.get_lpips.cache_clear()
    gt, pr = _pair("render", 3, 64, 80, seed=9)
    v = metrics.compute_lpips(gt, pr)
    assert v.shape == (3,) and not v.requires_grad
    assert metrics.get_lpips(DEV) is metrics.get_lpips(DEV)
    m = pl.LPIPS(weights=SD).to(DEV)
    assert torch.equal(v, m(gt, pr, normalize=True).detach()[:, 0, 0, 0])
    metrics.get_lpips.cache_clear()


def test_render_to_loss_chain_matches_the_oracle_image_gradient():
    """decoder_forward -> photometric_loss + 0.1 LPIPS on color[:, 1:-1] -> backward to the Gaussians, against the same
    chain fed dL/dcolor from the fp64 oracle (and, for the bound, from PyTorch's TF32 sequence)."""
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
    model = pl.LPIPS(weights=SD).to(DEV)

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
    for tag, dtype, tf32 in (("fp64", torch.float64, False), ("torch_tf32", torch.float32, True)):
        _, dl, _ = _torch(x, y, True, dout, dtype, tf32)
        dcolor = torch.zeros_like(color)
        dcolor[:, 1:-1] = (dphoto + dl.double()).reshape(b, v - 2, 3, *hw).float().to(DEV)
        leaves_o = [t.clone().requires_grad_(True) for t in base]
        color_o, _ = decoder_forward(*leaves_o, ext, intr, nr, fr, hw, bg)
        color_o.backward(dcolor)
        grads[tag] = (dcolor, [t.grad for t in leaves_o])
    ref_c, ref_l = grads["fp64"]
    tf_c, tf_l = grads["torch_tf32"]
    rc, rc_t = _rel(color.grad.double(), ref_c.double()), _rel(tf_c.double(), ref_c.double())
    print(f"[lpips] chain dL/dcolor rel-L2 ours {rc:.2e}, torch_tf32 {rc_t:.2e}")
    assert rc <= max(2 * rc_t, 1e-3)
    for name, ours, ref, tf in zip(("means", "covariances", "harmonics", "opacities"), leaves, ref_l, tf_l):
        r, r_t = _rel(ours.grad.double(), ref.double()), _rel(tf.double(), ref.double())
        print(f"[lpips] chain dL/d{name} rel-L2 ours {r:.2e}, torch_tf32 {r_t:.2e}")
        assert r <= max(2 * r_t, 1e-3), name
