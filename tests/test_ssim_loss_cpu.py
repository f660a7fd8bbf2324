"""CPU checks of the photometric training loss: the fp64 oracle (oracle/ssim_loss_oracle.py) against the reference's own
loss code (tests/golden/ssim_loss.npz, recorded by tests/golden/make_ssim_loss_golden.py and re-run live when
$PF3PLAT_ROOT names a PF3plat checkout), closed forms, the C ABI's struct layout and argument checks, and the Python
entry points' input handling.  No device is needed."""
import ctypes
import importlib.util
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import ssim_loss_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ssim_loss.npz")
CASES = ("random", "render", "identical", "out_of_range", "tiny_5x7", "tiny_1x1", "batch_37x45")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def _oracle_case(z, name, window):
    x, y, w = z[f"{name}/x"], z[f"{name}/y"], z[f"{name}/w_img"]
    s, m, gx, gy = so.per_image_with_grads(x, y, d_ssim=w, window=window)
    return {"ssim_img": s.numpy(), "ssim_mean": s.mean().numpy(), "grad_x": gx.numpy(), "grad_y": gy.numpy(),
            "loss_mse": m.mean().numpy(), "loss_multissim": (1 - s.mean()).numpy()}


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_reference_fp64_fixture(golden, name):
    ours = _oracle_case(golden, name, so.reference_window())
    for k, a in ours.items():
        b = golden[f"{name}/f64/{k}"]
        tol = 1e-10 * np.abs(b).max() + 1e-15   # the identical pair's gradients are rounding noise around 0
        assert np.abs(a - b).max() <= tol, (name, k, np.abs(a - b).max(), tol)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_reference_fp32_fixture(golden, name):
    ours = _oracle_case(golden, name, so.reference_window())
    worst = {k: float(np.abs(a - golden[f"{name}/f32/{k}"]).max()) for k, a in ours.items()}
    print(f"[ssim-loss] {name} fp32 reference vs fp64 oracle: {worst}")
    assert max(worst.values()) <= 2e-6, worst


def test_exact_window_differs_from_the_reference_window_only_by_its_float32_rounding(golden):
    """The kernels use the exact (separable) window rounded once to float32; the reference rounds its taps, their
    normalisation and their outer product to float32.  The difference is far below the GPU tolerance (1e-5)."""
    ref = so.reference_window()
    exact = torch.outer(so.gaussian_taps(), so.gaussian_taps())
    assert float((ref - exact).abs().max()) < 1e-8
    for name in CASES:
        a = _oracle_case(golden, name, None)["ssim_img"]
        assert np.abs(a - golden[f"{name}/f64/ssim_img"]).max() < 1e-6, name


def test_the_reference_reruns_live_and_agrees_with_the_fixture(golden):
    if not os.environ.get("PF3PLAT_ROOT"):
        pytest.skip("PF3PLAT_ROOT is not set: the reference module cannot be rerun")
    spec = importlib.util.spec_from_file_location("make_ssim_loss_golden",
                                                  os.path.join(ROOT, "tests", "golden", "make_ssim_loss_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    ms, mse_mod = gen.load_reference_losses()
    for name in CASES:
        x = torch.from_numpy(golden[f"{name}/x"]).double()
        y = torch.from_numpy(golden[f"{name}/y"]).double()
        w = torch.from_numpy(golden[f"{name}/w_img"])
        for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
            out = gen.run_reference(ms, mse_mod, x, y, w, dt)
            for k, v in out.items():
                b = golden[f"{name}/{tag}/{k}"]
                tol = (1e-12 if tag == "f64" else 1e-6) * np.abs(b).max() + 1e-15
                assert np.abs(v.numpy() - b).max() <= tol, (name, tag, k)


@pytest.mark.parametrize("shape", [(2, 3, 16, 16), (1, 1, 1, 1), (1, 2, 5, 7), (2, 1, 13, 4)])
def test_identical_images_give_one_and_zero_gradient(shape):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    s_map = so.ssim_map(x, x)
    assert float((s_map - 1).abs().max()) < 1e-14
    dx, dy = so.closed_form_backward(x, x, torch.ones(shape[0]))
    _, _, gx, gy = so.per_image_with_grads(x, x, d_ssim=torch.ones(shape[0]))
    for g in (dx, dy, gx, gy):
        assert float(g.abs().max()) < 1e-12


def _window_mass(h, w):
    """W(p): the mass of the 11x11 window that falls inside an h x w image when centred on p."""
    g = so.gaussian_taps().numpy()
    mass = lambda n: np.array([sum(g[k] for k in range(11) if 0 <= i + k - 5 < n) for i in range(n)])
    return np.outer(mass(h), mass(w))


@pytest.mark.parametrize("hw", [(1, 1), (5, 7), (12, 30), (40, 1)])
def test_a_constant_image_has_the_closed_form_moments(hw):
    h, w = hw
    c = 0.37
    x = torch.full((1, 1, h, w), c, dtype=torch.float64)
    y = torch.rand((1, 1, h, w), generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    ux, _, vx, _, _ = so.moments(x, y)
    W = _window_mass(h, w)
    np.testing.assert_allclose(ux[0, 0].numpy(), c * W, rtol=1e-13, atol=0)
    np.testing.assert_allclose(vx[0, 0].numpy(), c * c * W * (1 - W), rtol=1e-10, atol=1e-16)


@pytest.mark.parametrize("shape", [(2, 3, 24, 20), (1, 1, 1, 1), (2, 3, 5, 7), (1, 2, 11, 11), (1, 1, 12, 30), (1, 1, 40, 1)])
def test_closed_form_backward_equals_autograd(shape):
    g = torch.Generator().manual_seed(5)
    x = -0.1 + 1.3 * torch.rand(shape, generator=g, dtype=torch.float64)
    y = torch.rand(shape, generator=g, dtype=torch.float64)
    ds, dm = torch.randn(shape[0], generator=g, dtype=torch.float64), torch.randn(shape[0], generator=g, dtype=torch.float64)
    dx, dy = so.closed_form_backward(x, y, ds, dm)
    _, _, gx, gy = so.per_image_with_grads(x, y, d_ssim=ds, d_mse=dm)
    scale = float(gx.abs().max())
    assert float((dx - gx).abs().max()) <= 3e-15 * max(scale, 1.0)
    assert float((dy - gy).abs().max()) <= 3e-15 * max(scale, 1.0)


@pytest.mark.parametrize("shape", [(1, 2, 6, 9), (1, 1, 1, 1), (1, 1, 5, 7)])
def test_closed_form_backward_equals_finite_differences(shape):
    g = torch.Generator().manual_seed(6)
    x = torch.rand(shape, generator=g, dtype=torch.float64)
    y = torch.rand(shape, generator=g, dtype=torch.float64)
    ds, dm = torch.tensor([0.7], dtype=torch.float64), torch.tensor([-1.3], dtype=torch.float64)
    dx, dy = so.closed_form_backward(x, y, ds, dm)
    loss = lambda a, b: float((ds * so.ssim_per_image(a, b)).sum() + (dm * so.mse_per_image(a, b)).sum())
    h = 1e-6
    flat = np.random.default_rng(0).choice(x.numel(), size=min(8, x.numel()), replace=False)
    for i in flat:
        for t, d in ((0, dx), (1, dy)):
            p, m = [x.clone(), y.clone()], [x.clone(), y.clone()]
            p[t].view(-1)[i] += h
            m[t].view(-1)[i] -= h
            fd = (loss(*p) - loss(*m)) / (2 * h)
            assert abs(fd - float(d.view(-1)[i])) <= 1e-7 * max(1.0, abs(fd)), (i, t, fd, float(d.view(-1)[i]))


def test_loss_config_layout_matches_the_header(capi, tmp_path):
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %zu %zu\\n", sizeof(GsLossConfig), offsetof(GsLossConfig, pred_stride),'
                    ' offsetof(GsLossConfig, gt_stride), offsetof(GsLossConfig, with_mse));return 0;}')
    exe = tmp_path / "sizes"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    size, o_ps, o_gs, o_mse = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    C = capi.GsLossConfig
    assert (ctypes.sizeof(C), C.pred_stride.offset, C.gt_stride.offset, C.with_mse.offset) == (size, o_ps, o_gs, o_mse)


def test_null_and_invalid_arguments_are_rejected_without_a_device(capi):
    L = capi.lib()
    byref = ctypes.byref
    cfg = capi.GsLossConfig(batch=2, channels=3, height=256, width=256, pred_stride=3 * 256 * 256,
                            gt_stride=3 * 256 * 256, with_mse=1)
    assert L.gs_photometric_scratch_bytes(byref(cfg)) == 2 * 8 * 2 * 3 * 64
    tiny = capi.GsLossConfig(batch=1, channels=1, height=1, width=1, pred_stride=0, gt_stride=0, with_mse=0)
    assert L.gs_photometric_scratch_bytes(byref(tiny)) == 2 * 8           # a 1 x 1 image is legal: one tile
    assert L.gs_photometric_scratch_bytes(None) == -1
    fake = 4096  # never dereferenced: every check below fails (or returns) before the device is touched
    assert L.gs_photometric_forward(None, fake, fake, fake, fake, fake, None) == -1
    assert L.gs_photometric_backward(None, fake, fake, fake, fake, fake, fake, None, None) == -1
    assert L.gs_photometric_forward(byref(cfg), None, fake, fake, fake, fake, None) == -1
    assert L.gs_photometric_forward(byref(cfg), fake, fake, None, fake, fake, None) == -1      # no scratch
    assert L.gs_photometric_forward(byref(cfg), fake, fake, fake, fake, None, None) == -1      # with_mse, no out_mse
    assert L.gs_photometric_forward(byref(cfg), fake, fake, fake + 4, fake, fake, None) == -1  # misaligned scratch
    assert b"aligned" in L.gs_last_error()
    assert L.gs_photometric_backward(byref(cfg), None, fake, fake, fake, fake, fake, None, None) == -1
    for field, value in (("height", 0), ("width", -3), ("channels", 0), ("batch", -1), ("with_mse", 2),
                         ("pred_stride", 3 * 256 * 256 - 1), ("gt_stride", 0)):
        bad = capi.GsLossConfig.from_buffer_copy(cfg)
        setattr(bad, field, value)
        assert L.gs_photometric_scratch_bytes(byref(bad)) == -1, field
        assert L.gs_photometric_forward(byref(bad), fake, fake, fake, fake, fake, None) == -1, field
        assert L.gs_photometric_backward(byref(bad), fake, fake, fake, fake, fake, fake, None, None) == -1, field
    empty = capi.GsLossConfig.from_buffer_copy(cfg)
    empty.batch = 0
    assert L.gs_photometric_forward(byref(empty), fake, fake, fake, fake, fake, None) == 0
    assert L.gs_photometric_backward(byref(empty), fake, fake, fake, fake, fake, fake, None, None) == 0


def test_python_entry_points_refuse_what_they_cannot_run():
    from pf3plat_b200 import losses
    x = torch.rand(2, 3, 16, 16)
    with pytest.raises(ValueError, match="window_size"):
        losses.ssim(x, x, window_size=7)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        losses.ssim(x, x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        losses.photometric_loss(x, x)
    with pytest.raises(ValueError, match="same"):
        losses.ssim(x, x[:1])
    with pytest.raises(ValueError):
        losses.ssim(x[0], x[0])


def test_views_whose_batch_dimensions_collapse_are_read_in_place():
    from pf3plat_b200.losses import _layout
    chw = 3 * 8 * 10
    color = torch.rand(1, 5, 3, 8, 10)
    t, n, _, stride = _layout(color[:, 1:-1])
    assert t.data_ptr() == color[:, 1:-1].data_ptr() and n == 3 and stride == chw
    color = torch.rand(4, 3, 3, 8, 10)                        # PF3plat's training shape: one inner view per scene
    t, n, _, stride = _layout(color[:, 1:-1])
    assert t.data_ptr() == color[:, 1].data_ptr() and n == 4 and stride == 3 * chw
    color = torch.rand(2, 5, 3, 8, 10)                        # 2 x 3 inner views do not collapse to one stride
    t, n, _, stride = _layout(color[:, 1:-1])
    assert t.is_contiguous() and t.data_ptr() != color.data_ptr() and n == 6 and stride == chw
    t, _, _, _ = _layout(torch.rand(2, 3, 8, 10).transpose(-1, -2))   # a non-contiguous (c, h, w) block is copied
    assert t.is_contiguous()
    t, n, _, _ = _layout(torch.rand(1, 3, 8, 10).expand(4, 3, 8, 10))  # stride 0 between images: copied
    assert t.is_contiguous() and n == 4
