"""GPU tests of the plane-sweep cost volume (pf3plat_b200.costvolume.plane_sweep_cost_volume -> csrc/gs_costvolume.cu)
against the fp64 oracle (tests/costvolume_oracle.py), the reference's own functions recorded in
tests/golden/costvolume.npz, and the reference's op sequence restated below in float32 with F.grid_sample."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pf3plat_b200.costvolume import plane_sweep_cost_volume
from tests import costvolume_oracle as O
from tests.test_costvolume_cpu import CASES

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
VALUE_RTOL, GRAD_RTOL, FLOOR = 1e-4, 1e-3, 1e-5


def worst_ratio(got, want, rtol, what):
    """max over elements of |got - want| / max(rtol |want|, FLOOR max|want|); the non-finite elements must match."""
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    assert got.shape == want.shape, what
    assert torch.equal(torch.isnan(got), torch.isnan(want)), f"{what}: NaN pattern differs"
    inf = torch.isinf(want)
    assert torch.equal(torch.isinf(got), inf) and torch.equal(got[inf], want[inf]), f"{what}: Inf pattern differs"
    fin = torch.isfinite(want)
    if not fin.any():
        return 0.0
    g, w = got[fin], want[fin]
    bound = torch.maximum(rtol * w.abs(), torch.full_like(w, FLOOR * float(w.abs().max())))
    bound = torch.where(bound > 0, bound, torch.full_like(w, 1e-30))
    return float(((g - w).abs() / bound).max())


def run(features, K, E, near, far, D, cot, deterministic=False):
    f = features.detach().clone().requires_grad_(True) if features.is_contiguous() else features
    torch.use_deterministic_algorithms(deterministic)
    try:
        cost = plane_sweep_cost_volume(f, K, E, near, far, D)
        (grad,) = torch.autograd.grad(cost, f, cot)
    finally:
        torch.use_deterministic_algorithms(False)
    return cost.detach(), grad


def golden_inputs(case):
    t = lambda k: torch.tensor(case[k], dtype=torch.float32, device=DEV)
    return t("features"), t("intrinsics"), t("extrinsics"), t("near"), t("far"), int(case["D"]), t("cotangent")


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_cases(name, deterministic):
    case = CASES[name]
    cost, grad = run(*golden_inputs(case), deterministic=deterministic)
    if deterministic:  # the exact accumulators turn an infinite gradient term into NaN (DESIGN.md 5.11)
        fin = np.isfinite(case["grad64"])
        assert torch.equal(torch.isfinite(grad).cpu(), torch.from_numpy(fin))
        g64 = torch.where(torch.from_numpy(fin), torch.from_numpy(case["grad64"]), grad.double().cpu())
        g32 = torch.where(torch.from_numpy(fin), torch.from_numpy(case["grad32"]).double(), grad.double().cpu())
    else:
        g64, g32 = case["grad64"], case["grad32"]
    r = [worst_ratio(cost, case["value64"], VALUE_RTOL, "value vs fp64"),
         worst_ratio(cost, case["value32"], VALUE_RTOL, "value vs fp32"),
         worst_ratio(grad, g64, GRAD_RTOL, "grad vs fp64"), worst_ratio(grad, g32, GRAD_RTOL, "grad vs fp32")]
    print(f"{name} det={deterministic}: worst ratios value {r[0]:.3f} / {r[1]:.3f}, grad {r[2]:.3f} / {r[3]:.3f}")
    assert max(r) <= 1.0, r


# ---- the reference's op sequence (depth_predictor_multiview.py:91-141, :28-88, :309-343), restated in float32 ----

def reference_ops(features, intrinsics, extrinsics, near, far, D):
    b, v, c, h, w = features.shape
    vb = lambda t: t.transpose(0, 1).reshape(v * b, *t.shape[2:])
    feat01 = vb(features)
    if v == 2:
        pose = extrinsics[:, 1].inverse() @ extrinsics[:, 0]
        poses = [torch.cat((pose, pose.inverse()), dim=0)]
    else:
        poses = [torch.cat([extrinsics[:, (i + s) % v].inverse() @ extrinsics[:, i] for i in range(v)], dim=0)
                 for s in range(1, v)]
    K = intrinsics[:, :, :3, :3].clone().detach()
    K[:, :, 0, :] *= float(w)
    K[:, :, 1, :] *= float(h)
    K = vb(K)
    lo, hi = vb(1.0 / far.detach())[:, None], vb(1.0 / near.detach())[:, None]
    depth = (1.0 / (lo + torch.linspace(0.0, 1.0, D, device=lo.device)[None] * (hi - lo)))[:, :, None, None]
    depth = depth.repeat(1, 1, h, w)
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    grid = torch.stack([xs, ys, torch.ones_like(xs)]).float().to(features.device).reshape(1, 3, -1).repeat(v * b, 1, 1)
    out = []
    for s, pose in enumerate(poses, start=1):
        with torch.no_grad():
            pts = torch.inverse(K).bmm(grid)
            pts = torch.bmm(pose[:, :3, :3], pts).unsqueeze(2).repeat(1, 1, D, 1) * depth.view(v * b, 1, D, h * w)
            pts = pts + pose[:, :3, -1:].unsqueeze(-1)
            pts = torch.bmm(K, pts.view(v * b, 3, -1)).view(v * b, 3, D, h * w)
            px = pts[:, :2] / pts[:, -1:].clamp(min=1e-3)
            g = torch.stack([2 * px[:, 0] / (w - 1) - 1, 2 * px[:, 1] / (h - 1) - 1], dim=-1)
        feat10 = vb(features[:, [(i + s) % v for i in range(v)]])
        warped = F.grid_sample(feat10, g.view(v * b, D * h, w, 2), mode="bilinear", padding_mode="zeros",
                               align_corners=True).view(v * b, c, D, h, w)
        out.append((feat01.unsqueeze(2) * warped).sum(1) / (c ** 0.5))
    return torch.mean(torch.stack(out, dim=0), dim=0)


def seeded_case(b, v, C, h, w, D, seed):
    """Spatially smooth features (bilinearly upsampled 8x8 noise plus a little pixel noise), cameras a short baseline
    apart looking at the depth range, per-(scene, view) near and far."""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.randn(b * v, C, 8, 8, generator=g)
    f = F.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=False) + 0.1 * torch.randn(b * v, C, h, w, generator=g)
    E = torch.eye(4).repeat(b, v, 1, 1)
    for i in range(b):
        for j in range(1, v):
            a = torch.randn(3, generator=g) * 0.05
            Kx = torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
            E[i, j, :3, :3] = torch.matrix_exp(Kx)
            E[i, j, :3, 3] = torch.randn(3, generator=g) * 0.15
    K = torch.zeros(b, v, 3, 3)
    K[..., 0, 0] = 0.9 + 0.2 * torch.rand(b, v, generator=g)
    K[..., 1, 1] = 0.9 + 0.2 * torch.rand(b, v, generator=g)
    K[..., 0, 2] = 0.5 + 0.02 * torch.randn(b, v, generator=g)
    K[..., 1, 2] = 0.5 + 0.02 * torch.randn(b, v, generator=g)
    K[..., 2, 2] = 1.0
    near = 0.5 + 0.5 * torch.rand(b, v, generator=g)
    far = 20.0 + 10.0 * torch.rand(b, v, generator=g)
    cot = torch.randn(v * b, D, h, w, generator=g)
    to = lambda t: t.to(DEV)
    return to(f.reshape(b, v, C, h, w)), to(K), to(E), to(near), to(far), D, to(cot)


SHAPES = {"train_b14_v2": (14, 2, 256, 64, 64, 32), "v3_b4": (4, 3, 128, 48, 40, 16)}


def oracle_per_scene(f, K, E, near, far, D, cot):
    """the fp64 oracle, one scene at a time (a scene's cost and gradient depend on its own views only)"""
    b, v = f.shape[:2]
    value = torch.empty(v * b, D, *f.shape[-2:], dtype=torch.float64, device=f.device)
    grad = torch.empty(f.shape, dtype=torch.float64, device=f.device)
    for i in range(b):
        fo = f[i:i + 1].double().requires_grad_(True)
        oc = O.cost_volume(fo, K[i:i + 1].double(), E[i:i + 1].double(), near[i:i + 1].double(), far[i:i + 1].double(), D)
        rows = [vi * b + i for vi in range(v)]
        (go,) = torch.autograd.grad(oc, fo, cot[rows].double())
        value[rows], grad[i:i + 1] = oc.detach(), go
    return value, grad


def ratio_beyond_reference_error(got, ref32, oracle, rtol):
    """worst |got - ref32| / (bound + |ref32 - oracle|): the float32 op sequence is itself off the exact value by more
    than the bound at the training shape (its pixel coordinates are rounded to float32 at up to 64 px), so a kernel is
    held to lie within the bound of the reference plus the reference's own error"""
    got, ref32, oracle = got.double(), ref32.double(), oracle.double()
    assert torch.equal(torch.isfinite(got), torch.isfinite(ref32))
    bound = torch.clamp(rtol * ref32.abs(), min=FLOOR * float(ref32.abs().max()))
    return float(((got - ref32).abs() / (bound + (ref32 - oracle).abs())).max())


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_seeded_shapes_against_reference_ops_and_oracle(shape):
    b, v, C, h, w, D = SHAPES[shape]
    f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=len(shape))
    cost, grad = run(f, K, E, near, far, D, cot)
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    r = [worst_ratio(cost, ov, VALUE_RTOL, "value vs oracle"), worst_ratio(grad, og, GRAD_RTOL, "grad vs oracle")]
    fr = f.detach().clone().requires_grad_(True)
    ref = reference_ops(fr, K, E, near, far, D)
    (gref,) = torch.autograd.grad(ref, fr, cot)
    ref = ref.detach()
    own = [worst_ratio(ref, ov, VALUE_RTOL, "fp32 ops vs oracle"), worst_ratio(gref, og, GRAD_RTOL, "fp32 ops vs oracle")]
    r += [ratio_beyond_reference_error(cost, ref, ov, VALUE_RTOL), ratio_beyond_reference_error(grad, gref, og, GRAD_RTOL)]
    print(f"{shape}: worst ratios vs oracle: value {r[0]:.3f}, grad {r[1]:.3f}; vs the fp32 ops beyond their own error: "
          f"value {r[2]:.3f}, grad {r[3]:.3f}; the fp32 ops vs oracle: value {own[0]:.3f}, grad {own[1]:.3f}")
    assert max(r) <= 1.0, r


def test_deterministic_mode_is_bit_reproducible_and_agrees_with_the_default():
    b, v, C, h, w, D = SHAPES["train_b14_v2"]
    f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=3)
    c1, g1 = run(f, K, E, near, far, D, cot, deterministic=True)
    c2, g2 = run(f, K, E, near, far, D, cot, deterministic=True)
    c0, g0 = run(f, K, E, near, far, D, cot)
    assert torch.equal(c1, c2) and torch.equal(g1, g2) and torch.equal(c0, c1)
    assert worst_ratio(g0, g1, GRAD_RTOL, "default vs deterministic") <= 1.0
    # a cotangent on view 1's rows only: view 1's gradient is then the feat01 role alone (every source-role term that
    # reaches it is zero), view 0's the source role alone
    cot1 = cot.clone()
    cot1[:b] = 0
    for det in (False, True):
        ga = run(f, K, E, near, far, D, cot1, deterministic=det)[1]
        gb = run(f, K, E, near, far, D, cot1, deterministic=det)[1]
        assert torch.equal(ga[:, 1], gb[:, 1]), det
        assert ga[:, 1].abs().sum() > 0 and ga[:, 0].abs().sum() > 0


def test_cameras_get_no_gradient_and_the_drop_in_matches():
    b, v, C, h, w, D = SHAPES["train_b14_v2"]
    f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=5)
    leaves = [t.clone().requires_grad_(True) for t in (f, K, E, near, far)]
    features, intrinsics, extrinsics, n, fa = leaves
    # the drop-in of INTEGRATION.md 4, against the restated reference lines
    cost = plane_sweep_cost_volume(features, intrinsics, extrinsics, n, fa, D)
    feat01 = features.transpose(0, 1).reshape(v * b, C, h, w)
    raw = torch.cat((cost, feat01), dim=1)
    with torch.no_grad():
        ref = torch.cat((reference_ops(f, K, E, near, far, D), f.transpose(0, 1).reshape(v * b, C, h, w)), dim=1)
    assert worst_ratio(raw.detach(), ref, VALUE_RTOL, "raw_correlation_in") <= 1.0
    raw.backward(torch.randn_like(raw))
    assert features.grad is not None
    assert all(t.grad is None for t in (intrinsics, extrinsics, n, fa))


def test_no_sync_side_stream_and_non_contiguous_features():
    b, v, C, h, w, D = 3, 3, 40, 24, 20, 8
    f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=9)
    c_ref, g_ref = run(f, K, E, near, far, D, cot)
    # the features as a strided view of a channel-last tensor, 4x4 intrinsics
    base = f.permute(0, 1, 3, 4, 2).contiguous().requires_grad_(True)
    nc = base.permute(0, 1, 4, 2, 3)
    assert not nc.is_contiguous()
    K4 = torch.eye(4, device=DEV).repeat(b, v, 1, 1)
    K4[..., :3, :3] = K
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            cost = plane_sweep_cost_volume(nc, K4, E, near, far, D)
            (g,) = torch.autograd.grad(cost, base, cot)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(cost, c_ref)
    assert worst_ratio(g.permute(0, 1, 4, 2, 3), g_ref, GRAD_RTOL, "non-contiguous") <= 1.0


def test_bad_arguments_raise_before_any_launch():
    f = torch.randn(1, 2, 4, 5, 6, device=DEV)
    K, E = torch.eye(3, device=DEV).repeat(1, 2, 1, 1), torch.eye(4, device=DEV).repeat(1, 2, 1, 1)
    n, fa = torch.ones(1, 2, device=DEV), torch.full((1, 2), 5.0, device=DEV)
    with pytest.raises(ValueError):
        plane_sweep_cost_volume(f[:, :1], K[:, :1], E[:, :1], n[:, :1], fa[:, :1], 4)  # v < 2
    with pytest.raises(ValueError):
        plane_sweep_cost_volume(f[..., :1, :], K, E, n, fa, 4)  # h < 2
    with pytest.raises(ValueError):
        plane_sweep_cost_volume(f, K[:, :, :2], E, n, fa, 4)  # mismatched shapes
    with pytest.raises(TypeError):
        plane_sweep_cost_volume(f.double(), K, E, n, fa, 4)
    with pytest.raises(RuntimeError):
        plane_sweep_cost_volume(f.cpu(), K, E, n, fa, 4)
    assert math.isfinite(float(plane_sweep_cost_volume(f, K, E, n, fa, 4).sum()))
