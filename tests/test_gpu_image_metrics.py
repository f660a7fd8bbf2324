"""GPU tests of the image-side kernels -- PSNR and SSIM (csrc/gs_metrics.cu), LPIPS-VGG (csrc/gs_lpips.cu) and the
photometric loss (csrc/gs_losses.cu) -- on non-finite images and on the shapes and layouts where a streaming or tiled
kernel goes wrong, against plain fp64 restatements of the same operations.

Non-finite images follow the reference: PSNR clips with torch.clip, which keeps NaN, so an image holding a NaN scores
NaN (a +-Inf pixel is clipped and stays finite); SSIM, LPIPS and the loss do not clip, so NaN and +-Inf give NaN.
Entries are NaN exactly where the fp64 oracle's are, gradients are non-finite exactly where the oracle's are (the
oracle run on the GPU, as PyTorch's CUDA ops propagate NaN; the CPU run is reported beside it), and the clean images
of a poisoned batch get the bits of a batch of the clean images alone.

Tolerances are those of the suites these kernels already have: PSNR 1e-4 dB, SSIM 2e-5 absolute, LPIPS the TF32-relative
bound of tests/test_gpu_lpips.py, the loss VALUE_TOL and check_grad of tests/test_gpu_losses.py.
"""
import pytest
import torch

from oracle import lpips_oracle as lo
from oracle import ssim_loss_oracle as so
from oracle import ssim_oracle
from pf3plat_b200 import losses
from pf3plat_b200 import lpips as pl
from pf3plat_b200.metrics import compute_psnr, compute_ssim
from tests.util import check_grad

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PSNR_TOL = 1e-4
SSIM_TOL = 2e-5
LOSS_VALUE_TOL = 1e-5
SD = lo.random_state_dict(11)


# ---------------------------------------------------------------------------------------------------------------------
# oracles and comparisons
# ---------------------------------------------------------------------------------------------------------------------
def psnr_oracle(gt, pr):
    """The reference's compute_psnr in fp64: -10 log10(mean((clip(gt) - clip(pr))^2)) with torch.clip (keeps NaN)."""
    gt, pr = gt.detach().cpu().double().clip(0, 1), pr.detach().cpu().double().clip(0, 1)
    return -10 * ((gt - pr) ** 2).flatten(1).mean(1).log10()


def ssim_oracle_of(gt, pr):
    return torch.from_numpy(ssim_oracle.compute_ssim(gt.detach().cpu().double().numpy(), pr.detach().cpu().double().numpy()))


def assert_values(label, got, want, tol):
    """NaN exactly where `want` is NaN, +-inf exactly where it is, the finite entries within `tol` (a tensor or float)."""
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    assert got.shape == want.shape, (label, got.shape, want.shape)
    nan_got, nan_want = torch.isnan(got), torch.isnan(want)
    print(f"[image-metrics] {label}: NaN at {nan_want.nonzero().flatten().tolist()} (oracle), "
          f"{nan_got.nonzero().flatten().tolist()} (ours); values {got.numpy()[:6]}")
    assert torch.equal(nan_got, nan_want), (label, got, want)
    inf = torch.isinf(want)
    assert torch.equal(torch.isinf(got), inf) and torch.equal(got[inf], want[inf]), (label, got, want)
    fin = torch.isfinite(want)
    err = (got[fin] - want[fin]).abs()
    bound = tol[fin] if torch.is_tensor(tol) else tol
    assert bool((err <= bound).all()), (label, float(err.max()) if err.numel() else 0.0, got, want)


def assert_nonfinite_sets(label, got, want, cpu=None):
    """The non-finite elements of `got` are exactly those of `want` (PyTorch's CUDA run); `cpu` (the same oracle on the
    CPU) is reported beside it."""
    bad_got, bad_want = ~torch.isfinite(got), ~torch.isfinite(want)
    extra = f", CPU oracle {'agrees' if torch.equal(~torch.isfinite(cpu), bad_want) else 'DIFFERS'}" if cpu is not None else ""
    print(f"[image-metrics] {label}: {int(bad_want.sum())} of {want.numel()} gradient elements non-finite (oracle), "
          f"{int(bad_got.sum())} (ours), {int((bad_got != bad_want).sum())} differ{extra}")
    assert torch.equal(bad_got, bad_want), label


# ---------------------------------------------------------------------------------------------------------------------
# poisoned batches: (image, which input, channel, row, column, value); a row or column of None poisons the whole image
# ---------------------------------------------------------------------------------------------------------------------
NAN, INF = float("nan"), float("inf")


def _spots(h, w):
    return {"corner": (0, 0), "edge": (h - 1, w // 2), "interior": (h // 2, w // 3), "far_corner": (h - 1, w - 1),
            "left_edge": (h // 3, 0)}


def poison_plan(layout, c, h, w):
    """-> (poisons, clean image indices, batch size).  `which` is "x" (prediction / in0), "y" (ground truth / in1) or
    "xy" (both); poisons of a channel the images do not have are left out."""
    plan, clean, n = _poison_plan(layout, h, w)
    return [p for p in plan if p[2] is None or p[2] < c], clean, n


def _poison_plan(layout, h, w):
    s = _spots(h, w)
    if layout == "a":  # NaN in one input or both, at a corner, an edge and inside; +Inf
        plan = [(1, "x", 0, *s["corner"], NAN), (3, "y", 1, *s["edge"], NAN), (4, "xy", 2, *s["interior"], NAN),
                (5, "x", 1, *s["left_edge"], INF)]
        return plan, [0, 2], 6
    if layout == "b":  # -Inf, a whole NaN image, +-Inf in both
        plan = [(0, "y", 2, *s["far_corner"], -INF), (2, "x", None, None, None, NAN), (3, "y", 0, *s["edge"], INF),
                (3, "x", 1, *s["interior"], -INF)]
        return plan, [1, 4], 5
    raise KeyError(layout)


def apply_poison(x, y, plan):
    x, y = x.clone(), y.clone()
    for img, which, c, r, col, v in plan:
        for t, name in ((x, "x"), (y, "y")):
            if name in which:
                if c is None:
                    t[img] = v
                else:
                    t[img, c, r, col] = v
    return x, y


def _rand_pair(n, c, h, w, seed, lo_=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (lo_ + (hi - lo_) * torch.rand(n, c, h, w, generator=g), lo_ + (hi - lo_) * torch.rand(n, c, h, w, generator=g))


# ---------------------------------------------------------------------------------------------------------------------
# PSNR
# ---------------------------------------------------------------------------------------------------------------------
# c*h*w is a multiple of 4 here, so every image of a fresh allocation takes the 16-byte path and a sub-batch of the clean
# images has the summation order of the full batch
@pytest.mark.parametrize("layout", ["a", "b"])
@pytest.mark.parametrize("c,h,w", [(3, 32, 48), (1, 17, 20)])
def test_psnr_of_non_finite_images(layout, c, h, w):
    plan, clean, n = poison_plan(layout, c, h, w)
    gt, pr = apply_poison(*_rand_pair(n, c, h, w, seed=h * w + n, lo_=-0.2, hi=1.2), plan)
    got = compute_psnr(gt.to(DEV), pr.to(DEV))
    want = psnr_oracle(gt, pr)
    assert bool(torch.isnan(want).any()) and bool(torch.isfinite(want).any())
    assert_values(f"psnr {layout} {n}x{c}x{h}x{w}", got, want, PSNR_TOL)
    alone = compute_psnr(gt[clean].to(DEV), pr[clean].to(DEV))
    assert torch.equal(got[clean], alone)


PSNR_SHAPES = [  # (batch, c, h, w): c*h*w mod 4 = 0..3; n below, at and above 65 536 (where the 64-block grid-stride
    # loop starts to iterate), up to 3 x 512^2; batches 1, 14 and 60
    (2, 1, 1, 4), (3, 1, 1, 5), (2, 1, 2, 3), (3, 1, 1, 7), (5, 3, 37, 53), (4, 3, 17, 130), (2, 1, 1, 1), (2, 1, 1, 3),
    (2, 1, 256, 256), (2, 1, 1, 65540), (3, 1, 1, 65537), (2, 1, 1, 65538), (2, 1, 1, 65539), (2, 3, 150, 151),
    (1, 3, 512, 512), (14, 3, 256, 256), (60, 3, 64, 64), (60, 3, 33, 47),
]


@pytest.mark.parametrize("b,c,h,w", PSNR_SHAPES)
def test_psnr_shapes(b, c, h, w):
    gt, pr = _rand_pair(b, c, h, w, seed=b * 7 + c * h * w, lo_=-0.3, hi=1.3)   # clipped on both sides
    got = compute_psnr(gt.to(DEV), pr.to(DEV))
    assert got.dtype == torch.float32 and got.shape == (b,)
    assert_values(f"psnr {b}x{c}x{h}x{w}", got, psnr_oracle(gt, pr), PSNR_TOL)


@pytest.mark.parametrize("c,h,w", [(3, 64, 80), (3, 37, 53), (1, 1, 5)])
def test_psnr_of_a_prediction_only_4_byte_aligned(c, h, w):
    """A prediction sliced at a storage offset of one float: contiguous, but not 16-byte aligned, so the kernel reads
    it (and the aligned ground truth beside it) with scalar loads."""
    b = 3
    n = c * h * w
    g = torch.Generator().manual_seed(n)
    buf = torch.rand(b * n + 4, generator=g).to(DEV)
    pr = buf[1:1 + b * n].view(b, c, h, w)
    gt = torch.rand(b, c, h, w, generator=g).to(DEV)
    assert pr.is_contiguous() and pr.data_ptr() % 16 == 4
    got = compute_psnr(gt, pr)
    assert_values(f"psnr misaligned {b}x{c}x{h}x{w}", got, psnr_oracle(gt, pr), PSNR_TOL)
    assert_values(f"psnr misaligned {b}x{c}x{h}x{w} vs copy", got, compute_psnr(gt, pr.clone()), PSNR_TOL)


def test_psnr_of_the_references_call_forms_equals_its_contiguous_copy():
    """rgb_gt[1:-1] and rearrange(x[:, 1:-1], "b v c h w -> (b v) c h w") as the reference evaluates them."""
    g = torch.Generator().manual_seed(21)
    views = torch.rand(5, 3, 64, 80, generator=g).to(DEV)
    pred = torch.rand(5, 3, 64, 80, generator=g).to(DEV)
    a = compute_psnr(views[1:-1], pred[1:-1])
    assert torch.equal(a, compute_psnr(views[1:-1].contiguous().clone(), pred[1:-1].contiguous().clone()))
    assert_values("psnr rgb_gt[1:-1]", a, psnr_oracle(views[1:-1], pred[1:-1]), PSNR_TOL)
    for b in (1, 3):
        x = torch.rand(b, 5, 3, 64, 80, generator=g).to(DEV)
        y = torch.rand(b, 5, 3, 64, 80, generator=g).to(DEV)
        fx, fy = x[:, 1:-1].reshape(-1, 3, 64, 80), y[:, 1:-1].reshape(-1, 3, 64, 80)   # einops' rearrange is this view
        got = compute_psnr(fy, fx)
        assert torch.equal(got, compute_psnr(fy.contiguous().clone(), fx.contiguous().clone()))
        assert_values(f"psnr rearrange b={b}", got, psnr_oracle(fy, fx), PSNR_TOL)


def test_psnr_edges():
    g = torch.Generator().manual_seed(22)
    x = torch.rand(4, 3, 33, 47, generator=g)
    # identical images: mse 0, PSNR +inf as the reference's log10(0) gives
    same = compute_psnr(x.to(DEV), x.to(DEV))
    assert bool(torch.isposinf(same).all()), same
    # +-Inf and values far outside [0, 1] are clipped
    y = torch.rand(4, 3, 33, 47, generator=g)
    y[0, 0, 0, 0], y[1, 2, 32, 46], y[2, 1, 16, 0] = INF, -INF, 1e30
    y[3] = -5.0
    assert_values("psnr clipped infinities", compute_psnr(x.to(DEV), y.to(DEV)), psnr_oracle(x, y), PSNR_TOL)
    # mse near 1e-12: PSNR near 120 dB
    base = 0.25 + 0.5 * torch.rand(3, 3, 64, 64, generator=g)
    sign = torch.where(torch.rand(3, 3, 64, 64, generator=g) < 0.5, -1.0, 1.0)
    near = base + 1e-6 * sign
    want = psnr_oracle(base, near)
    assert bool((want > 115).all() and (want < 125).all()), want
    assert_values("psnr near 120 dB", compute_psnr(base.to(DEV), near.to(DEV)), want, PSNR_TOL)


def test_psnr_dtype_follows_the_inputs():
    g = torch.Generator().manual_seed(23)
    x, y = torch.rand(3, 3, 20, 24, generator=g, dtype=torch.float64), torch.rand(3, 3, 20, 24, generator=g, dtype=torch.float64)
    got = compute_psnr(x.to(DEV), y.to(DEV))
    assert got.dtype == torch.float64
    assert_values("psnr fp64 inputs", got, psnr_oracle(x.float(), y.float()), PSNR_TOL)
    assert compute_psnr(x.half().to(DEV), y.half().to(DEV)).dtype == torch.float16
    assert compute_psnr(x.to(DEV), y.float().to(DEV)).dtype == torch.float64


def test_psnr_on_a_side_stream_gives_the_bits_of_the_default_stream():
    x, y = (t.to(DEV) for t in _rand_pair(14, 3, 256, 256, seed=24))
    ref = compute_psnr(x, y)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        got = compute_psnr(x, y)
    side.synchronize()
    assert torch.equal(got, ref)


def test_psnr_of_more_images_than_a_grid_dimension_holds():
    """70 000 images of 1 x 1 x 4: more than the 65 535 blocks of gridDim.y, so the batch is launched in chunks."""
    g = torch.Generator().manual_seed(25)
    x, y = torch.rand(70000, 1, 1, 4, generator=g), torch.rand(70000, 1, 1, 4, generator=g)
    x[69999, 0, 0, 1] = NAN
    got = compute_psnr(x.to(DEV), y.to(DEV))
    assert_values("psnr 70000 images", got, psnr_oracle(x, y), PSNR_TOL)
    assert torch.equal(got[65530:65540], compute_psnr(x[65530:65540].to(DEV), y[65530:65540].to(DEV)))


# ---------------------------------------------------------------------------------------------------------------------
# SSIM
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["a", "b"])
@pytest.mark.parametrize("c,h,w", [(3, 32, 48), (1, 17, 20), (4, 11, 11)])
def test_ssim_of_non_finite_images(layout, c, h, w):
    plan, clean, n = poison_plan(layout, c, h, w)
    gt, pr = apply_poison(*_rand_pair(n, c, h, w, seed=h * w + n + 1), plan)
    got = compute_ssim(gt.to(DEV), pr.to(DEV))
    want = ssim_oracle_of(gt, pr)
    assert bool(torch.isnan(want).any()) and bool(torch.isfinite(want).any())
    assert_values(f"ssim {layout} {n}x{c}x{h}x{w}", got, want, SSIM_TOL)
    assert torch.equal(got[clean], compute_ssim(gt[clean].to(DEV), pr[clean].to(DEV)))


def _structured(b, c, h, w, seed, lo_=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(b, c, h, w, generator=g)
    ys, xs = torch.meshgrid(torch.linspace(0, 6.28, h), torch.linspace(0, 6.28, w), indexing="ij")
    gt = 0.5 * gt + 0.25 * (1 + torch.sin(3 * xs) * torch.cos(2 * ys))
    pred = gt + 0.1 * torch.randn(b, c, h, w, generator=g)
    return lo_ + (hi - lo_) * gt, lo_ + (hi - lo_) * pred


CROPS = (1, 31, 32, 33, 64, 65)   # H - 10 and W - 10: the 32 x 32 tile's edge on both sides of the crop


@pytest.mark.parametrize("ch", CROPS)
def test_ssim_crop_extents(ch):
    for k, cw in enumerate(CROPS):
        c = (1, 3, 4)[k % 3]
        gt, pr = _structured(2, c, ch + 10, cw + 10, seed=ch * 100 + cw)
        assert_values(f"ssim crop {ch}x{cw} c={c}", compute_ssim(gt.to(DEV), pr.to(DEV)), ssim_oracle_of(gt, pr), SSIM_TOL)


@pytest.mark.parametrize("b,c,h,w,lo_,hi", [(60, 3, 256, 256, 0.0, 1.0), (3, 1, 40, 70, -0.4, 1.5), (2, 4, 75, 43, -0.3, 1.3),
                                            (3, 3, 37, 53, 0.0, 1.0)])
def test_ssim_shapes_and_values_outside_the_unit_range(b, c, h, w, lo_, hi):
    gt, pr = _structured(b, c, h, w, seed=b + c + h + w, lo_=lo_, hi=hi)   # SSIM does not clip
    assert_values(f"ssim {b}x{c}x{h}x{w} in [{lo_}, {hi}]", compute_ssim(gt.to(DEV), pr.to(DEV)), ssim_oracle_of(gt, pr),
                  SSIM_TOL)


def test_ssim_of_constant_and_identical_images():
    vals = [(0.25, 0.75), (0.0, 1.0), (0.5, 0.5), (1.0, 0.0), (0.125, 0.1875)]
    gt = torch.stack([torch.full((3, 24, 30), a) for a, _ in vals])
    pr = torch.stack([torch.full((3, 24, 30), b) for _, b in vals])
    c1 = 0.01 ** 2
    closed = torch.tensor([(2 * a * b + c1) / (a * a + b * b + c1) for a, b in vals], dtype=torch.float64)
    got = compute_ssim(gt.to(DEV), pr.to(DEV))
    # the variances vanish: a moment that cancels to a spurious fp32 variance (~1e-7 a^2, against C2 = 9e-4) shows here
    print(f"[image-metrics] ssim constant images: |ours - closed form| {(got.cpu().double() - closed).abs().numpy()}")
    assert_values("ssim constant images (closed form)", got, closed, SSIM_TOL)
    assert_values("ssim constant images (oracle)", got, ssim_oracle_of(gt, pr), SSIM_TOL)
    # a flat bright region beside a textured one, and a smooth ramp: the same cancellation at a smaller scale
    g = torch.Generator().manual_seed(30)
    flat = torch.full((2, 3, 60, 70), 0.9)
    flat[:, :, :, 35:] = torch.rand(2, 3, 60, 35, generator=g)
    ramp = torch.linspace(0.6, 0.95, 70).expand(2, 3, 60, 70).clone()
    for label, x, y in (("flat + texture", flat, flat * 0.97 + 0.02), ("ramp", ramp, ramp.flip(-1))):
        assert_values(f"ssim {label}", compute_ssim(x.to(DEV), y.to(DEV)), ssim_oracle_of(x, y), SSIM_TOL)
    x, _ = _structured(4, 3, 45, 61, seed=31)
    same = compute_ssim(x.to(DEV), x.to(DEV))
    assert torch.equal(ssim_oracle_of(x, x), torch.ones(4, dtype=torch.float64))
    assert torch.equal(same, torch.ones(4, device=DEV)), same   # as the reference: exactly 1


def test_ssim_of_fp64_and_fp16_inputs():
    gt, pr = _structured(3, 3, 40, 52, seed=32)
    for dtype in (torch.float64, torch.float16):
        a, b = gt.to(dtype), pr.clamp(0, 1).to(dtype)
        got = compute_ssim(a.to(DEV), b.to(DEV))
        assert got.dtype == dtype
        want = ssim_oracle_of(a, b)   # the oracle reads the very values the kernel gets
        half_ulp = (want.abs() * 2.0 ** -11) if dtype == torch.float16 else 0.0   # the result is rounded to fp16
        assert_values(f"ssim {dtype}", got, want, SSIM_TOL + half_ulp)


def test_ssim_of_strided_and_misaligned_layouts():
    g = torch.Generator().manual_seed(33)
    views = torch.rand(5, 3, 40, 52, generator=g).to(DEV)
    pred = (views + 0.1 * torch.randn(5, 3, 40, 52, generator=g).to(DEV)).clamp(0, 1)
    a = compute_ssim(views[1:-1], pred[1:-1])
    assert torch.equal(a, compute_ssim(views[1:-1].clone(), pred[1:-1].clone()))
    assert_values("ssim rgb_gt[1:-1]", a, ssim_oracle_of(views[1:-1], pred[1:-1]), SSIM_TOL)
    for b in (1, 3):
        x = torch.rand(b, 5, 3, 40, 52, generator=g).to(DEV)
        y = (x + 0.1 * torch.randn(b, 5, 3, 40, 52, generator=g).to(DEV)).clamp(0, 1)
        fx, fy = x[:, 1:-1].reshape(-1, 3, 40, 52), y[:, 1:-1].reshape(-1, 3, 40, 52)
        got = compute_ssim(fx, fy)
        assert torch.equal(got, compute_ssim(fx.clone(), fy.clone()))
        assert_values(f"ssim rearrange b={b}", got, ssim_oracle_of(fx, fy), SSIM_TOL)
    n = 3 * 3 * 37 * 53
    buf = torch.rand(n + 4, generator=g).to(DEV)
    pr = buf[1:1 + n].view(3, 3, 37, 53)
    gt = torch.rand(3, 3, 37, 53, generator=g).to(DEV)
    assert pr.data_ptr() % 16 == 4
    got = compute_ssim(gt, pr)
    assert torch.equal(got, compute_ssim(gt, pr.clone()))
    assert_values("ssim misaligned", got, ssim_oracle_of(gt, pr), SSIM_TOL)


def test_ssim_of_more_images_than_a_grid_dimension_holds():
    """65 537 images of 1 x 11 x 11: more than the 65 535 blocks of gridDim.z, so the batch is launched in chunks.  The
    images repeat 7 patterns; each pattern's value is checked against the oracle and every copy must have its bits."""
    base_gt, base_pr = _structured(7, 1, 11, 11, seed=34)
    base_gt[6, 0, 5, 5] = NAN
    idx = torch.arange(65537) % 7
    got = compute_ssim(base_gt[idx].to(DEV), base_pr[idx].to(DEV))
    small = compute_ssim(base_gt.to(DEV), base_pr.to(DEV))
    assert_values("ssim 7 patterns", small, ssim_oracle_of(base_gt, base_pr), SSIM_TOL)
    assert bool(torch.isnan(small[6])) and torch.equal(got.isnan(), small.isnan()[idx.to(DEV)])
    assert torch.equal(got.nan_to_num(-7.0), small.nan_to_num(-7.0)[idx.to(DEV)])


# ---------------------------------------------------------------------------------------------------------------------
# photometric loss
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["a", "b"])
@pytest.mark.parametrize("c,h,w", [(3, 32, 48), (1, 17, 20), (3, 5, 7)])
def test_loss_of_non_finite_images(layout, c, h, w):
    plan, clean, n = poison_plan(layout, c, h, w)
    x, y = apply_poison(*_rand_pair(n, c, h, w, seed=h * w + n + 2), plan)   # x = prediction, y = ground truth
    g = torch.Generator().manual_seed(n + h)
    ws, wm = torch.randn(n, generator=g), torch.randn(n, generator=g)
    xg, yg = x.to(DEV).requires_grad_(True), y.to(DEV).requires_grad_(True)
    s, m = losses._per_image(xg, yg)
    ((s * ws.to(DEV)).sum() + (m * wm.to(DEV)).sum()).backward()
    so_c, mo_c, gxo_c, gyo_c = so.per_image_with_grads(x, y, d_ssim=ws, d_mse=wm)
    so_g, mo_g, gxo_g, gyo_g = (t.cpu() for t in so.per_image_with_grads(x.to(DEV), y.to(DEV), d_ssim=ws.to(DEV),
                                                                          d_mse=wm.to(DEV)))
    label = f"loss {layout} {n}x{c}x{h}x{w}"
    assert bool(torch.isnan(so_g).any()) and bool(torch.isfinite(so_g).any())
    assert_values(f"{label} ssim", s, so_g, LOSS_VALUE_TOL)
    assert_values(f"{label} mse", m, mo_g, LOSS_VALUE_TOL)
    for name, ours, want, cpu in (("dL/dpred", xg.grad.cpu(), gxo_g, gxo_c), ("dL/dgt", yg.grad.cpu(), gyo_g, gyo_c)):
        assert_nonfinite_sets(f"{label} {name}", ours, want, cpu)
        fin = torch.isfinite(want)
        check_grad(f"{label} {name} (finite elements)", ours[fin], want[fin].numpy())
    # the clean images alone: the same bits, values and gradients
    xc, yc = x[clean].to(DEV).requires_grad_(True), y[clean].to(DEV).requires_grad_(True)
    sc, mc = losses._per_image(xc, yc)
    ((sc * ws[clean].to(DEV)).sum() + (mc * wm[clean].to(DEV)).sum()).backward()
    assert torch.equal(s.detach()[clean], sc.detach()) and torch.equal(m.detach()[clean], mc.detach())
    assert torch.equal(xg.grad[clean], xc.grad) and torch.equal(yg.grad[clean], yc.grad)


# ---------------------------------------------------------------------------------------------------------------------
# LPIPS
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    return pl.LPIPS(net="vgg", weights=SD).to(DEV)


def _torch_lpips(x0, x1, normalize, dout, dtype, tf32, device=DEV):
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        return lo.with_grads(x0, x1, SD, normalize, dout, device=device, dtype=dtype)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _ours_lpips(model, x0, x1, normalize, dout):
    a, b = x0.to(DEV).requires_grad_(True), x1.to(DEV).requires_grad_(True)
    v = model(a, b, normalize=normalize).reshape(-1)
    (v * dout.to(DEV)).sum().backward()
    return v.detach().cpu().double(), a.grad.cpu().double(), b.grad.cpu().double()


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def lpips_plan(n, h, w):
    """Poisons for an LPIPS batch of n images (n = 1: one poison per parametrisation); the bottom row is the row the
    floor pool drops when h is odd, the right column the column it drops when w is odd."""
    s = _spots(h, w)
    full = [(0, "x", 0, *s["corner"], NAN), (1, "y", 1, h - 1, w // 2, NAN), (2, "xy", 2, *s["interior"], NAN),
            (3, "x", 1, *s["left_edge"], INF), (4, "y", 0, h // 2, w - 1, -INF), (6, "x", None, None, None, NAN)]
    return [p for p in full if p[0] < n]


LPIPS_CASES = [  # (n, h, w, normalize, poison index for n = 1)
    (1, 16, 16, True, 0), (1, 16, 16, False, 1), (1, 16, 16, True, 3), (1, 16, 16, False, 4), (1, 16, 16, True, 5),
    (3, 17, 130, True, None), (3, 17, 130, False, None), (14, 256, 256, True, None), (14, 256, 256, False, None),
]


@pytest.mark.parametrize("n,h,w,normalize,single", LPIPS_CASES)
def test_lpips_of_non_finite_images(model, n, h, w, normalize, single):
    if single is not None:
        _, which, c, r, col, v = lpips_plan(7, h, w)[single]
        plan = [(0, which, c, r, col, v)]
    elif n == 3:   # a NaN in the row the floor pool drops (h = 17), a clean image, +Inf in the ground truth
        plan = [(0, "x", 1, h - 1, 7, NAN), (2, "y", 2, h // 2, w // 2, INF)]
    else:
        plan = lpips_plan(n, h, w)
    clean = [i for i in range(n) if i not in {p[0] for p in plan}]
    x0, x1 = apply_poison(*_rand_pair(n, 3, h, w, seed=h * w + n), plan)
    dout = 0.5 + torch.rand(n, generator=torch.Generator().manual_seed(n), dtype=torch.float64)
    v, g0, g1 = _ours_lpips(model, x0, x1, normalize, dout)
    v64, g064, g164 = _torch_lpips(x0, x1, normalize, dout, torch.float64, False)
    vt, gt0, gt1 = _torch_lpips(x0, x1, normalize, dout, torch.float32, True)
    cpu = _torch_lpips(x0, x1, normalize, dout, torch.float64, False, device="cpu") if h * w * n <= 3 * 17 * 130 else None
    label = f"lpips {n}x3x{h}x{w} normalize={normalize} poisons={plan}"
    assert bool(torch.isnan(v64).all()) if not clean else bool(torch.isnan(v64).any())
    if cpu is not None:
        print(f"[image-metrics] {label}: CPU oracle value NaN set "
              f"{'agrees' if torch.equal(torch.isnan(cpu[0]), torch.isnan(v64)) else 'DIFFERS'}")
    fin = torch.isfinite(v64)
    err_t = float((vt.double() - v64)[fin].abs().max()) if fin.any() else 0.0
    assert_values(f"{label} value", v, v64, torch.maximum(torch.full_like(v64, 2 * err_t), 1e-4 * v64.abs() + 1e-6))
    for k, (ours, want, tf, c) in enumerate(((g0, g064, gt0, cpu and cpu[1]), (g1, g164, gt1, cpu and cpu[2]))):
        assert_nonfinite_sets(f"{label} dL/din{k}", ours, want, c)
        m = torch.isfinite(want)
        if not m.any():
            continue
        mt = m & torch.isfinite(tf)
        rel, rel_t = _rel(ours[m], want[m]), _rel(tf.double()[mt], want[mt])
        print(f"[image-metrics] {label} dL/din{k} finite elements: rel-L2 ours {rel:.2e}, torch_tf32 {rel_t:.2e}")
        assert rel <= max(2 * rel_t, 1e-3), (rel, rel_t)
    if clean:
        vc, gc0, gc1 = _ours_lpips(model, x0[clean], x1[clean], normalize, dout[clean])
        assert torch.equal(v[clean], vc) and torch.equal(g0[clean], gc0) and torch.equal(g1[clean], gc1)
