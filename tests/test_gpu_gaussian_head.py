"""The Gaussian head's kernels (pf3plat_b200.gaussian_head, csrc/gs_gaussian_head.cu) against the reference's own fp64
record (tests/golden/gaussian_head.npz), the fp64 oracle (tests/gaussian_head_oracle.py) and the existing route on the
same device (the glue statements around pf3plat_b200.adapter.GaussianAdapter): values element-wise within
1e-5 (|ref| + 1), gradients within 1e-3 (|ref| + rms ref), with the same non-finite elements.  Cotangents of Gaussians
whose sigmoids lie within float32 rounding of saturation are zeroed, as tests/strict_parity.py does.  Also: bit-identical
reruns, side streams and scenes computed alone, the backward under deterministic algorithms, decoder_forward on both
routes, and the stretch from depth_update to a loss under sync debug mode "error"."""
import math

import numpy as np
import pytest
import torch

from pf3plat_b200.adapter import GaussianAdapterCfg
from tests import gaussian_head_oracle as O
from tests.gaussian_head_route import existing_route
from tests.test_gaussian_head_cpu import NAMES, Z, case, recorded

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
VAL_TOL, GRAD_TOL = 1e-5, 1e-3
KEYS = ("means", "covariances", "harmonics", "opacities")


def cfg_for(deg):
    return GaussianAdapterCfg(gaussian_scale_min=O.SCALE_MIN, gaussian_scale_max=O.SCALE_MAX, sh_degree=int(deg))


def value_ratio(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isfinite(got), np.isfinite(ref))
    f = np.isfinite(ref)
    return float((np.abs(got[f] - ref[f]) / (VAL_TOL * (np.abs(ref[f]) + 1.0))).max(initial=0.0))


def grad_ratio(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape and np.array_equal(np.isfinite(got), np.isfinite(ref))
    f = np.isfinite(ref)
    rms = math.sqrt(float((ref[f] ** 2).mean())) if f.any() else 0.0
    return float((np.abs(got[f] - ref[f]) / (GRAD_TOL * (np.abs(ref[f]) + rms) + 1e-30)).max(initial=0.0))


def fragile_mask(c):
    """[b, G]: Gaussians with a sigmoid argument beyond float32 saturation (|x| > 15), whose gradient float32 cannot
    carry; their cotangents are zeroed"""
    raw = np.asarray(c["raw"], np.float64)
    b = c["c2w"].shape[0]
    h, w = raw.shape[-2:]
    big = (np.abs(raw[:, :5]) > 15).any(1) | (np.abs(np.asarray(c["logits"], np.float64)[:, 1]) > 15)
    return big.reshape(2, b, h * w).transpose(1, 0, 2).reshape(b, 2 * h * w)


def masked_cotangents(c):
    keep = ~fragile_mask(c)
    cot = {}
    for k in KEYS:
        a = np.asarray(c["cot_" + k], np.float64)
        cot[k] = a * keep.reshape(keep.shape + (1,) * (a.ndim - 2))
    return cot


def run_head(c, cot=None, deterministic=False, stream=None):
    from pf3plat_b200.gaussian_head import gaussian_head
    t = {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV).requires_grad_(cot is not None)
         for k in O.INPUTS}
    K = torch.tensor(np.asarray(c["K"]), dtype=torch.float32, device=DEV)
    h, w = c["raw"].shape[-2:]
    g = gaussian_head(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(c["sh_degree"]), (h, w))
    vals = {k: getattr(g, k) for k in KEYS}
    grads = None
    if cot is not None:
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(deterministic)
        try:
            loss = sum((torch.tensor(cot[k], dtype=torch.float32, device=DEV) * vals[k]).sum() for k in KEYS)
            loss.backward()
        finally:
            torch.use_deterministic_algorithms(prev)
        grads = {k: t[k].grad for k in O.INPUTS}
    return vals, grads


def np_(d):
    return {k: v.detach().cpu().numpy() for k, v in d.items()}


@pytest.mark.parametrize("name", NAMES)
def test_matches_the_reference_record_and_the_oracle(name):
    c = case(name)
    cot = masked_cotangents(c)
    vals, grads = run_head(c, cot)
    vals, grads = np_(vals), np_(grads)
    ovals, ograds = O.run(c, cot)
    for k in KEYS:
        assert value_ratio(recorded(name, k, vals[k]), Z[f"{name}/{k}64"]) <= 1.0, k
        assert value_ratio(vals[k], ovals[k]) <= 1.0, k
    for k in O.INPUTS:
        assert grad_ratio(grads[k], ograds[k]) <= 1.0, k
    if not fragile_mask(c).any():  # the record's cotangents are unmasked
        _, full = run_head(c, {k: c["cot_" + k] for k in KEYS})
        for k, g in np_(full).items():
            assert grad_ratio(recorded(name, "d_" + k, g), Z[f"{name}/d_{k}64"]) <= 1.0, k
    # exact zeros where the reference gives none: delta_disps, middle views, row 3 of c2w
    b, V = c["c2w"].shape[:2]
    assert (grads["logits"][:, 0] == 0).all()
    assert (grads["depths"].reshape(b, V, -1)[:, 1:V - 1] == 0).all()
    assert (grads["c2w"][:, 1:V - 1] == 0).all() and (grads["c2w"][:, :, 3] == 0).all()


def seeded(b, V, h, w, deg, seed=0):
    from tests.golden.make_gaussian_head_golden import make_case
    return make_case(seed, b, V, h, w, deg)


@pytest.mark.parametrize("b,V,h,w,deg", [(2, 3, 16, 24, 4), (1, 2, 33, 17, 3), (3, 5, 8, 9, 4), (2, 2, 128, 1, 2)])
def test_seeded_shapes_match_the_oracle_and_the_existing_route(b, V, h, w, deg):
    c = seeded(b, V, h, w, deg, seed=b * 100 + h)
    cot = masked_cotangents(c)
    vals, grads = run_head(c, cot)
    ovals, ograds = O.run(c, cot)
    for k in KEYS:
        assert value_ratio(vals[k].detach().cpu().numpy(), ovals[k]) <= 1.0, k
    for k in O.INPUTS:
        assert grad_ratio(grads[k].cpu().numpy(), ograds[k]) <= 1.0, k
    # the existing route on the same device, forward and backward
    t = {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV).requires_grad_(True) for k in O.INPUTS}
    K = torch.tensor(np.asarray(c["K"]), dtype=torch.float32, device=DEV)
    outs = existing_route(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(deg), h, w)
    sum((torch.tensor(cot[k], dtype=torch.float32, device=DEV) * o).sum() for k, o in zip(KEYS, outs)).backward()
    for k, o in zip(KEYS, outs):
        assert value_ratio(vals[k].detach().cpu().numpy(), o.detach().cpu().numpy()) <= 1.0, k
    for k in O.INPUTS:
        assert grad_ratio(grads[k].cpu().numpy(), t[k].grad.cpu().numpy()) <= 1.0, k
    assert vals["harmonics"].transpose(-1, -2).is_contiguous()


def test_bit_identical_reruns_side_streams_scenes_alone_and_deterministic_mode():
    c = seeded(3, 3, 20, 30, 4, seed=7)
    cot = masked_cotangents(c)
    v0, g0 = run_head(c, cot)
    v1, g1 = run_head(c, cot, deterministic=True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        v2, g2 = run_head(c, cot)
    torch.cuda.synchronize()
    for a, bb in ((v0, v1), (v0, v2), (g0, g1), (g0, g2)):
        for k in a:
            assert torch.equal(a[k], bb[k]), k
    V, hw = 3, 20 * 30
    for bi in range(3):
        one = {k: c[k][bi:bi + 1] for k in ("c2w", "K")}
        one.update(sh_degree=c["sh_degree"], depths=c["depths"][bi * V:(bi + 1) * V],
                   raw=c["raw"][[bi, 3 + bi]], logits=c["logits"][[bi, 3 + bi]])
        vo, go = run_head(one, {k: cot[k][bi:bi + 1] for k in KEYS})
        for k in KEYS:
            assert torch.equal(vo[k], v0[k][bi:bi + 1]), k
        assert torch.equal(go["c2w"], g0["c2w"][bi:bi + 1])
        assert torch.equal(go["depths"], g0["depths"][bi * V:(bi + 1) * V])
        assert torch.equal(go["raw"], g0["raw"][[bi, 3 + bi]]) and torch.equal(go["logits"], g0["logits"][[bi, 3 + bi]])
    assert hw > 128  # several CTAs per camera: the fixed-order finalize is exercised


def test_decoder_forward_on_both_routes():
    from pf3plat_b200.render import decoder_forward
    b, V, h, w, deg = 1, 2, 32, 32, 3
    c = seeded(b, V, h, w, deg, seed=3)
    c["raw"][:, 2:5] -= 3.0  # small Gaussians
    vals, _ = run_head(c)
    t = {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV) for k in O.INPUTS}
    K = torch.tensor(np.asarray(c["K"]), dtype=torch.float32, device=DEV)
    outs = existing_route(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(deg), h, w)
    ext = t["c2w"].clone()
    ext[:, :, :3, 3] -= 3.0 * ext[:, :, :3, 2]  # step back so that the Gaussians lie in front
    near, far = torch.full((b, V), 0.5, device=DEV), torch.full((b, V), 100.0, device=DEV)
    bg = torch.zeros(3, device=DEV)
    ours = decoder_forward(vals["means"], vals["covariances"], vals["harmonics"], vals["opacities"], ext, K, near, far,
                           (h, w), bg)[0]
    theirs = decoder_forward(*outs, ext, K, near, far, (h, w), bg)[0]
    assert torch.isfinite(ours).all()
    assert float((ours - theirs).abs().max()) <= 1e-3


def test_the_stretch_runs_without_a_host_synchronisation():
    from pf3plat_b200.encoder_depth import depth_update
    from pf3plat_b200.gaussian_head import gaussian_head
    from pf3plat_b200.poses import refine_poses
    b, V, h, w, deg, grid = 2, 3, 32, 32, 4, (8, 8)
    g = torch.Generator(device=DEV).manual_seed(0)
    near = 0.5 + torch.rand((b, V), generator=g, device=DEV)
    far = near + 50.0
    depth = (0.2 + torch.rand((b * V, 1, h, w), generator=g, device=DEV)) * 20.0
    ss0 = torch.randn((b, V, grid[0] * grid[1], 2), generator=g, device=DEV)
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]], device=DEV).expand(b, V, 3, 3).contiguous()
    enc0 = torch.zeros((b, V, 9), device=DEV)
    enc0[..., 0] = 1.0
    enc0[..., 4] = 1.0
    enc0[..., 6:] = torch.randn((b, V, 3), generator=g, device=DEV)
    delta0 = 0.05 * torch.randn((b, V, 9), generator=g, device=DEV)
    gamma0 = torch.ones(1, device=DEV)
    raw0 = torch.randn((2 * b, 9 + 3 * 25, h, w), generator=g, device=DEV)
    logits0 = torch.randn((2 * b, 2, h, w), generator=g, device=DEV)
    cfg = cfg_for(deg)

    def run(check):
        ss = ss0.clone().requires_grad_(True)
        enc = enc0.clone().requires_grad_(True)
        raw = raw0.clone().requires_grad_(True)
        logits = logits0.clone().requires_grad_(True)
        if check:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            depths, _ = depth_update(depth, ss, K, near, far, grid)
            _, c2w = refine_poses(enc, delta0, gamma0)
            gs = gaussian_head(raw, logits, depths, c2w, K, cfg, (h, w))
            loss = gs.means.square().mean() + gs.covariances.mean() + gs.harmonics.square().mean() + gs.opacities.mean()
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        return ss.grad, enc.grad, raw.grad, logits.grad

    run(False)  # warm up: library load, the SH fit tables, the masks
    grads = run(True)
    for gr in grads:
        assert torch.isfinite(gr).all() and gr.abs().sum() > 0


def test_inputs_are_refused():
    from pf3plat_b200.gaussian_head import gaussian_head
    b, V, h, w = 1, 3, 4, 5
    raw = torch.zeros(2 * b, 9 + 3 * 9, h, w, device=DEV)
    lg = torch.zeros(2 * b, 2, h, w, device=DEV)
    dp = torch.ones(b * V, 1, h, w, device=DEV)
    c2w = torch.eye(4, device=DEV).repeat(b, V, 1, 1)
    K = torch.eye(3, device=DEV).repeat(b, V, 1, 1)
    cfg = cfg_for(2)
    gaussian_head(raw, lg, dp, c2w, K, cfg, (h, w))
    with pytest.raises(TypeError, match="float32"):
        gaussian_head(raw.double(), lg, dp, c2w, K, cfg, (h, w))
    with pytest.raises(TypeError, match="CUDA"):
        gaussian_head(raw, lg, dp.cpu(), c2w, K, cfg, (h, w))
    with pytest.raises(ValueError, match="channels"):
        gaussian_head(raw[:, :-1], lg, dp, c2w, K, cfg, (h, w))
    with pytest.raises(ValueError, match="sh_degree"):
        gaussian_head(raw, lg, dp, c2w, K, cfg_for(5), (h, w))
    with pytest.raises(ValueError, match="depth-predictor views"):
        gaussian_head(torch.cat([raw, raw[:1]]), lg, dp, c2w, K, cfg, (h, w))
    with pytest.raises(ValueError, match="gaussians_per_pixel"):
        gaussian_head(raw, lg, dp, c2w, K, cfg, (h, w), gaussians_per_pixel=2)
    with pytest.raises(ValueError, match="gaussians_per_pixel"):
        gaussian_head(raw, lg, dp, c2w, K, cfg, (h, w), num_surfaces=2)
    with pytest.raises(ValueError, match="depths"):
        gaussian_head(raw, lg, dp[:, :, :, :-1], c2w, K, cfg, (h, w))
    with pytest.raises(ValueError, match="intrinsics"):
        gaussian_head(raw, lg, dp, c2w, K[:, :2], cfg, (h, w))
    with pytest.raises(ValueError, match="V >= 2"):
        gaussian_head(raw, lg, dp[:1], c2w[:, :1], K[:, :1], cfg, (h, w))
    with pytest.raises(ValueError, match="density_logits"):
        gaussian_head(raw, lg[:, :1], dp, c2w, K, cfg, (h, w))
    with pytest.raises(ValueError, match="must not require grad"):
        gaussian_head(raw, lg, dp, c2w, K.clone().requires_grad_(True), cfg, (h, w))
